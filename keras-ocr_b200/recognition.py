"""Recognizer: drop-in for ``keras_ocr.recognition.Recognizer`` (reference recognition.py:353-537)."""
import math
import string
import typing

import numpy as np
import torch

from . import _lib, tools, weights as weights_mod

DEFAULT_ALPHABET = string.digits + string.ascii_lowercase      # reference recognition.py:25
TARGET_HEIGHT, TARGET_WIDTH, STEPS = 31, 200, 48                # DEFAULT_BUILD_PARAMS, recognition.py:13-23
DEFAULT_BUILD_PARAMS = {"height": 31, "width": 200, "color": False, "filters": (64, 128, 256, 256, 512, 512, 512),
                        "rnn_units": (128, 128), "dropout": 0.25, "rnn_steps_to_discard": 2, "pool_size": 2}


def labels_to_text(rows, alphabet=DEFAULT_ALPHABET):
    """reference recognition.py:527-534: drop blank / -1, map indices to characters.

    Vectorised: the kept labels of all rows are gathered into ONE byte string with a newline after every row, decoded
    once and split (no per-character and no per-row Python work besides the split); alphabets that are not ASCII or
    contain a newline, and tables with out-of-range indices, take the reference's element-wise filter."""
    blank = len(alphabet)
    rows = np.asarray(rows)
    if rows.ndim == 2 and rows.size and alphabet.isascii() and "\n" not in alphabet:
        keep = (rows != blank) & (rows != -1)
        flat = rows[keep]
        if flat.size == 0 or (int(flat.min()) >= 0 and int(flat.max()) < blank):
            out = np.full(flat.size + rows.shape[0], 10, dtype=np.uint8)          # 10 = "\n"
            ends = np.cumsum(keep.sum(1) + 1) - 1
            chars = np.ones(out.size, dtype=bool)
            chars[ends] = False
            out[chars] = np.frombuffer(alphabet.encode("ascii"), dtype=np.uint8)[flat]
            return out.tobytes().decode("ascii").split("\n")[:-1]
    return ["".join(alphabet[idx] for idx in row if idx not in (blank, -1)) for row in rows]


def confidences(logp):
    """Word confidences exp(S) in (0, 1] (float32) from the greedy-path log-probabilities
    S = sum_t log(max_c p[t,c] + 1e-7) that ``b2o_crnn_forward_scored`` writes.  The 1e-7 floor lets S of a
    certain word reach 48 * log(1 + 1e-7) ~ 5e-6 > 0, hence the clip at 1."""
    return np.minimum(np.exp(np.asarray(logp, dtype=np.float32)), np.float32(1.0))


def check_beam(beam_width=None, top_paths=1):
    """Validates a decoder choice before anything is launched (``ValueError`` otherwise): ``beam_width=None`` is greedy
    CTC (the default, and then ``top_paths`` must be 1); an int 1 <= ``beam_width`` <= 128 is CTC prefix beam search
    (``b2o_crnn_forward_beam``) returning the ``top_paths`` best readings, 1 <= ``top_paths`` <= ``beam_width``."""
    def is_int(v):
        return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))
    if not is_int(top_paths) or top_paths < 1:
        raise ValueError(f"top_paths must be an int >= 1, got {top_paths!r}")
    if beam_width is None:
        if top_paths != 1:
            raise ValueError("top_paths > 1 needs beam search: pass beam_width")
        return
    if not is_int(beam_width) or not 1 <= beam_width <= _lib.MAX_BEAM_WIDTH:
        raise ValueError(f"beam_width must be None or an int in [1, {_lib.MAX_BEAM_WIDTH}], got {beam_width!r}")
    if top_paths > beam_width:
        raise ValueError(f"top_paths ({top_paths}) must not exceed beam_width ({beam_width})")


def _check_word(i, w, index, what):
    """The rules a lexicon entry and a training text share: a non-empty string of at most 48 characters of the
    alphabet (``index``: character -> label); ``ValueError`` naming entry ``i`` otherwise."""
    if not isinstance(w, str) or not w:
        raise ValueError(f"{what} {i} ({w!r}) is not a non-empty string")
    if len(w) > STEPS:
        raise ValueError(f"{what} {i} ({w!r}) is longer than {STEPS} characters")
    bad = next((ch for ch in w if ch not in index), None)
    if bad is not None:
        raise ValueError(f"{what} {i} ({w!r}) has {bad!r}, which is not in the alphabet")


def encode_csr(words, index):
    """Checked words -> CSR: (offsets (n+1) int32, labels int16), word i is labels[offsets[i]:offsets[i+1]]."""
    lengths = np.fromiter((len(w) for w in words), dtype=np.int64, count=len(words))
    offsets = np.zeros(len(words) + 1, np.int32)
    offsets[1:] = np.cumsum(lengths)
    labels = np.fromiter((index[ch] for w in words for ch in w), dtype=np.int16, count=int(lengths.sum()))
    return offsets, labels


def check_texts(texts, alphabet=DEFAULT_ALPHABET):
    """Validates the target texts of ``Recognizer.fit_top`` on the host, before anything is launched, and returns their
    CSR encoding (``encode_csr``).  The rules are the reference's training rules (``get_batch_generator``,
    recognition.py:440-449): every text is a non-empty string of at most 48 characters, all in ``alphabet``, without two
    spaces in a row; and it must be alignable in the 48 steps, i.e. its length plus its adjacent repeated characters
    (each needs a blank between its copies) is at most 48 -- Keras would give such a text an infinite loss and NaN
    gradients.  Texts may repeat.  ``ValueError`` names the first offending text."""
    if isinstance(texts, str) or not isinstance(texts, (list, tuple, np.ndarray)):
        raise ValueError("texts must be a list or tuple of strings")
    texts = list(texts)
    if not texts:
        raise ValueError("there are no texts")
    index = {ch: i for i, ch in enumerate(alphabet)}
    for i, w in enumerate(texts):
        _check_word(i, w, index, "text")
        if "  " in w:
            raise ValueError(f"text {i} ({w!r}) has two spaces in a row, which the reference does not train on")
        repeats = sum(a == b for a, b in zip(w, w[1:]))
        if len(w) + repeats > STEPS:
            raise ValueError(f"text {i} ({w!r}) cannot be aligned in {STEPS} steps: {len(w)} characters and {repeats} "
                             "doubled letters, each of which needs a blank")
    return encode_csr(texts, index)


class Lexicon:
    """A word list for lexicon-constrained decoding (``b2o_crnn_forward_lexicon``): every crop reads as the entry with the
    highest CTC forward log-probability -- the sum over every 48-step alignment that collapses to the entry -- and
    ``top_paths`` gives the P best entries.  Entries are non-empty strings over ``alphabet`` of at most 48 characters,
    distinct, at most 2^20 of them; anything else raises ``ValueError`` naming the first offending entry.  An entry whose
    doubled letters make it longer than 48 steps (length + adjacent repeats > 48) is valid but scores -inf.

    The lexicon is compiled once on the host (CSR: ``offsets`` (n+1) int32, ``labels`` int16) and uploaded lazily, once
    per CUDA device, so one object serves every rank of a sharded run.  A plain list or tuple of strings is accepted
    wherever a ``Lexicon`` is and is compiled for that call."""

    def __init__(self, words, alphabet=DEFAULT_ALPHABET):
        if isinstance(words, str) or not isinstance(words, (list, tuple)):
            raise ValueError("a lexicon is a list or tuple of strings")
        if not words:
            raise ValueError("the lexicon is empty")
        if len(words) > _lib.MAX_LEXICON_WORDS:
            raise ValueError(f"the lexicon has {len(words)} entries; at most {_lib.MAX_LEXICON_WORDS} are supported")
        index = {ch: i for i, ch in enumerate(alphabet)}
        seen = set()
        for i, w in enumerate(words):
            _check_word(i, w, index, "lexicon entry")
            if w in seen:
                raise ValueError(f"lexicon entry {i} ({w!r}) is a duplicate")
            seen.add(w)
        self.words, self.alphabet = tuple(words), alphabet
        lengths = np.fromiter((len(w) for w in words), dtype=np.int64, count=len(words))
        if lengths.sum() > _lib.MAX_LEXICON_LABELS:
            i = int(np.argmax(np.cumsum(lengths) > _lib.MAX_LEXICON_LABELS))
            raise ValueError(f"lexicon entry {i} ({words[i]!r}) takes the lexicon past {_lib.MAX_LEXICON_LABELS} "
                             "characters in all")
        self.offsets, self.labels = encode_csr(words, index)
        self._device = {}

    def __len__(self):
        return len(self.words)

    def device_arrays(self, device):
        """(offsets, labels) CUDA tensors on ``device``, uploaded on first use."""
        device = torch.device(device)
        if device not in self._device:
            self._device[device] = (torch.from_numpy(self.offsets).to(device), torch.from_numpy(self.labels).to(device))
        return self._device[device]


LM_BOS = 127                  # the code of <s> in a history (labels are < 126); </s> is label len(alphabet), the blank's
_LN10 = math.log(10.0)


class CharLM:
    """A character n-gram language model for CTC beam search (``b2o_crnn_forward_beam_lm``; DESIGN.md section 1,
    "Language model").  Symbols are the alphabet's labels, ``</s>`` (end of word) and ``<s>`` (start of word, only in
    histories); a word is the sentence ``<s> w </s>``.  A backoff model of order 2 <= N <= 8 with ARPA semantics:
    log P(w | h) = log P*(w | h) when (h, w) is listed, otherwise bo(h) + log P(w | h without its oldest symbol), bo(h) =
    0 for an unlisted h.  The tables are kept as ARPA stores them, in log10 (``logp10``, ``backoff10``: {tuple of
    symbols: value}, ``<s>`` = ``LM_BOS``, ``</s>`` = len(alphabet)), so ``to_arpa`` / ``from_arpa`` round-trip exactly;
    every score the package computes from them is a natural log.

    ``alpha`` (the weight of the model's log-probabilities) and ``beta`` (a bonus per character) are fixed at
    construction; ``weighted`` returns a copy with others that shares the tables.  The device form is uploaded lazily,
    once per CUDA device (``device_arrays``)."""

    ALPHA, BETA = 1.0, 2.0       # picked by scripts/bench_lm.py's sweep on its tuning pages (DESIGN.md section 5)

    def __init__(self, alphabet, order, logp10, backoff10, alpha=ALPHA, beta=BETA):
        if len(alphabet) > _lib.MAX_LM_CLASSES - 1:
            raise ValueError(f"a language model takes at most {_lib.MAX_LM_CLASSES - 1} alphabet characters, "
                             f"got {len(alphabet)}")
        if len(set(alphabet)) != len(alphabet):
            raise ValueError("the alphabet has repeated characters")
        if not 2 <= order <= _lib.MAX_LM_ORDER:
            raise ValueError(f"the order must be in [2, {_lib.MAX_LM_ORDER}], got {order}")
        eos = len(alphabet)
        missing = [s for s in range(eos + 1) if (s,) not in logp10]
        if missing:
            raise ValueError(f"no unigram for {self._token(alphabet, missing[0])!r}")
        self.alphabet, self.order = alphabet, int(order)
        self.logp10, self.backoff10 = logp10, backoff10
        self._histories = sorted(g for g in logp10 if len(g) < order and eos not in g)
        if len(self._histories) + 1 > _lib.MAX_LM_HISTORIES:
            raise ValueError(f"the model lists {len(self._histories) + 1} histories; at most {_lib.MAX_LM_HISTORIES} "
                             "are supported")
        self._check_weights(alpha, beta)
        self.alpha, self.beta = float(alpha), float(beta)
        self._tables = {}                 # shared by weighted copies: the host device form and its uploads per device

    @staticmethod
    def _check_weights(alpha, beta):
        for name, v in (("alpha", alpha), ("beta", beta)):
            ok = not isinstance(v, (bool, np.bool_)) and isinstance(v, (int, float, np.integer, np.floating))
            if ok:
                with np.errstate(over="ignore"):
                    ok = math.isfinite(float(np.float32(v)))         # the device takes them as float32
            if not ok:
                raise ValueError(f"{name} must be a number finite in float32, got {v!r}")

    @staticmethod
    def _token(alphabet, s):
        return "<s>" if s == LM_BOS else "</s>" if s == len(alphabet) else alphabet[s]

    def weighted(self, alpha=ALPHA, beta=BETA):
        """A copy with weights ``alpha`` and ``beta`` that shares this model's tables and device uploads."""
        self._check_weights(alpha, beta)
        other = object.__new__(CharLM)
        other.__dict__.update(self.__dict__)
        other.alpha, other.beta = float(alpha), float(beta)
        return other

    # ------------------------------------------------------------------ fitting
    @classmethod
    def fit(cls, words, alphabet=DEFAULT_ALPHABET, order=5, counts=None):
        """Interpolated Kneser-Ney of order ``order`` on ``words`` (checked as lexicon entries are; ``counts``: an
        optional positive int per word, its multiplicity).  One discount per order, D_n = n1 / (n1 + 2 n2) over that
        order's adjusted counts (0.5 when n1 or n2 is 0); the highest order and n-grams that begin with <s> count
        occurrences, the other orders continuation counts (distinct left neighbours); the unigrams interpolate with the
        uniform distribution over the alphabet and </s>.  Written in backoff form: P* = (c - D) / c(h) + gamma(h)
        P(w | h'), bo(h) = gamma(h).  fp64 with sorted iteration: the same input gives the same tables bit for bit."""
        if isinstance(words, str) or not isinstance(words, (list, tuple)):
            raise ValueError("words must be a list or tuple of strings")
        if not words:
            raise ValueError("there are no words")
        if not isinstance(order, (int, np.integer)) or isinstance(order, (bool, np.bool_)) \
                or not 2 <= order <= _lib.MAX_LM_ORDER:
            raise ValueError(f"the order must be an int in [2, {_lib.MAX_LM_ORDER}], got {order!r}")
        if len(alphabet) > _lib.MAX_LM_CLASSES - 1:
            raise ValueError(f"a language model takes at most {_lib.MAX_LM_CLASSES - 1} alphabet characters, "
                             f"got {len(alphabet)}")
        if counts is None:
            counts = [1] * len(words)
        if len(counts) != len(words) or any(isinstance(c, (bool, np.bool_)) or not isinstance(c, (int, np.integer))
                                            or c < 1 for c in counts):
            raise ValueError("counts must hold one positive int per word")
        index = {ch: i for i, ch in enumerate(alphabet)}
        for i, w in enumerate(words):
            _check_word(i, w, index, "word")
        n, eos = int(order), len(alphabet)
        raw = [None] + [dict() for _ in range(n)]          # raw[m][gram]: occurrences of the m-gram
        for w, c in zip(words, counts):
            seq = (LM_BOS,) + tuple(index[ch] for ch in w) + (eos,)
            for m in range(1, n + 1):
                table = raw[m]
                for i in range(len(seq) - m + 1):
                    g = seq[i:i + m]
                    table[g] = table.get(g, 0) + int(c)
        adj = [None] * (n + 1)                             # adjusted counts
        adj[n] = raw[n]
        for m in range(n - 1, 0, -1):
            left = {}
            for g in raw[m + 1]:
                left[g[1:]] = left.get(g[1:], 0) + 1
            adj[m] = {g: (c if g[0] == LM_BOS else left[g]) for g, c in raw[m].items()}
        adj[1].pop((LM_BOS,), None)                         # <s> is never predicted
        logp10, backoff10 = {}, {}
        prob = {}                                           # interpolated P(w | h) of listed (h, w), fp64
        vocab = eos + 1

        def lower(g):                                       # P(g[-1] | g[:-1]) by the backoff recursion, fp64
            if g in prob:
                return prob[g]
            return gamma.get(g[:-1], 1.0) * lower(g[1:])

        gamma = {}
        for m in range(1, n + 1):
            values = list(adj[m].values())
            n1, n2 = values.count(1), values.count(2)
            d = n1 / (n1 + 2.0 * n2) if n1 and n2 else 0.5
            by_h = {}
            for g in sorted(adj[m]):
                by_h.setdefault(g[:-1], []).append(g)
            for h in sorted(by_h):
                grams = by_h[h]
                total = float(sum(adj[m][g] for g in grams))
                gam = d * len(grams) / total
                if m == 1:
                    for s in range(vocab):
                        a = adj[1].get((s,), 0)
                        prob[(s,)] = max(a - d, 0.0) / total + gam / vocab
                else:
                    gamma[h] = gam
                    for g in grams:
                        prob[g] = (adj[m][g] - d) / total + gam * lower(g[1:])
        for g in sorted(prob):
            logp10[g] = math.log10(prob[g])
        logp10[(LM_BOS,)] = -99.0
        for h in sorted(gamma):
            backoff10[h] = math.log10(gamma[h])
        return cls(alphabet, n, logp10, backoff10)

    # ------------------------------------------------------------------ ARPA
    @classmethod
    def from_arpa(cls, path_or_text, alphabet=DEFAULT_ALPHABET):
        """A model from an ARPA file (a path, or the file's text): n-grams with <unk> are dropped; any other token
        outside the alphabet, <s> and </s>, a missing unigram, an order outside [2, 8], an n-gram whose history is not
        listed or a malformed line raise ``ValueError`` naming the line; so does a file whose sections do not hold the
        n-gram counts its header declares (<unk> lines included), or that lacks \\end\\, as a truncated file does.
        The alphabet may not contain whitespace (ARPA tokens are whitespace-separated).  Character-split text through KenLM's ``lmplz`` loads unchanged."""
        if any(ch.isspace() for ch in alphabet):
            raise ValueError("an alphabet with whitespace cannot be read from ARPA (its tokens are whitespace-separated)")
        text = path_or_text
        if "\n" not in path_or_text and not path_or_text.lstrip().startswith("\\data\\"):
            with open(path_or_text, encoding="utf-8") as f:
                text = f.read()
        index = {ch: i for i, ch in enumerate(alphabet)}
        index["<s>"], index["</s>"] = LM_BOS, len(alphabet)
        logp10, backoff10, declared, found = {}, {}, {}, {}
        m, seen_data, ended = 0, False, False
        for no, line in enumerate(text.splitlines(), 1):
            s = line.strip()
            if not s or ended:
                continue
            if s == "\\data\\":
                seen_data = True
                continue
            if s == "\\end\\":
                ended = True
                continue
            if not seen_data:
                continue
            if s.startswith("ngram ") and m == 0:
                try:
                    k, v = s[6:].split("=")
                    declared[int(k)] = int(v)
                except ValueError:
                    raise ValueError(f"line {no}: malformed count line {line!r}") from None
                continue
            if s.startswith("\\") and s.endswith("-grams:"):
                try:
                    m = int(s[1:-7])
                except ValueError:
                    raise ValueError(f"line {no}: malformed section header {line!r}") from None
                continue
            if m == 0:
                raise ValueError(f"line {no}: unexpected line {line!r}")
            f = s.split()
            found[m] = found.get(m, 0) + 1
            if len(f) not in (m + 1, m + 2):
                raise ValueError(f"line {no}: a {m}-gram line has {m + 1} or {m + 2} fields, got {line!r}")
            toks = f[1:m + 1]
            if "<unk>" in toks:
                continue
            try:
                vals = [float(f[0])] + ([float(f[m + 1])] if len(f) == m + 2 else [])
            except ValueError:
                raise ValueError(f"line {no}: malformed number in {line!r}") from None
            if not all(math.isfinite(v) for v in vals):
                raise ValueError(f"line {no}: non-finite value in {line!r}")
            bad = next((t for t in toks if t not in index), None)
            if bad is not None:
                raise ValueError(f"line {no}: token {bad!r} is not in the alphabet, <s> or </s>")
            g = tuple(index[t] for t in toks)
            if LM_BOS in g[1:] or len(alphabet) in g[:-1]:
                raise ValueError(f"line {no}: <s> may only open and </s> only close an n-gram: {line!r}")
            if m > 1 and g[:-1] not in logp10:
                raise ValueError(f"line {no}: the history of {line!r} is not listed")
            logp10[g] = vals[0]
            if len(vals) == 2 and vals[1] != 0.0:
                backoff10[g] = vals[1]
        if not seen_data:
            raise ValueError("no \\data\\ section")
        for k in sorted(set(declared) | set(found)):
            if declared.get(k, 0) != found.get(k, 0):
                raise ValueError(f"the header declares {declared.get(k, 0)} {k}-grams, the file holds {found.get(k, 0)}")
        if not ended:
            raise ValueError("no \\end\\ line: the file is truncated")
        order = max((len(g) for g in logp10), default=0)
        if not 2 <= order <= _lib.MAX_LM_ORDER:
            raise ValueError(f"the order must be in [2, {_lib.MAX_LM_ORDER}], got {order}")
        return cls(alphabet, order, logp10, backoff10)

    def to_arpa(self, path):
        """Writes the model as an ARPA file, 17 significant digits: ``from_arpa`` reads back the same tables."""
        grams = sorted(self.logp10, key=lambda g: (len(g), g))
        out = ["\\data\\"] + [f"ngram {m}={sum(len(g) == m for g in grams)}" for m in range(1, self.order + 1)]
        for m in range(1, self.order + 1):
            out += ["", f"\\{m}-grams:"]
            for g in grams:
                if len(g) == m:
                    toks = " ".join(self._token(self.alphabet, s) for s in g)
                    line = f"{self.logp10[g]:.17g}\t{toks}"
                    if g in self.backoff10:
                        line += f"\t{self.backoff10[g]:.17g}"
                    out.append(line)
        out += ["", "\\end\\", ""]
        with open(path, "w", encoding="utf-8") as f:
            f.write("\n".join(out))

    # ------------------------------------------------------------------ scores
    def log_prob(self, text):
        """The fp64 natural-log probability of the word ``text``, </s> included."""
        index = {ch: i for i, ch in enumerate(self.alphabet)}
        _check_word(0, text, index, "text")
        seq = (LM_BOS,) + tuple(index[ch] for ch in text) + (len(self.alphabet),)
        total = 0.0
        for i in range(1, len(seq)):
            total += self.logp_symbol(seq[i], seq[max(0, i - self.order + 1):i])
        return total

    def logp_symbol(self, w, h):
        """log P(w | h) (natural log, fp64) by the backoff recursion; ``h`` a tuple of symbols."""
        bo = 0.0
        h = tuple(h)[-(self.order - 1):] if self.order > 1 else ()
        while h + (w,) not in self.logp10:
            bo += self.backoff10.get(h, 0.0)
            h = h[1:]
        return (bo + self.logp10[h + (w,)]) * _LN10

    # ------------------------------------------------------------------ device form
    @staticmethod
    def history_key(h):
        """The uint64 key of history ``h``: (len << 56) | its symbols 8 bits each, oldest highest."""
        k = len(h) << 56
        for i, s in enumerate(h):
            k |= int(s) << (8 * (len(h) - 1 - i))
        return k

    def host_tables(self):
        """(keys (H,) uint64 sorted, rows (H, K) float32): every listed history, keys[0] = 0 the empty one; column
        c < K-1 log P(c | h) with the backoff folded in (fp64, rounded once), column K-1 log P(</s> | h)."""
        if "host" not in self._tables:
            k = len(self.alphabet) + 1
            hist = [()] + self._histories
            keys = np.array([self.history_key(h) for h in hist], np.uint64)
            order = np.argsort(keys, kind="stable")
            hist = [hist[i] for i in order]
            at = {h: i for i, h in enumerate(hist)}
            children = {}
            for g in self.logp10:
                children.setdefault(g[:-1], []).append(g)
            rows = np.empty((len(hist), k), np.float64)
            for h in sorted(hist, key=len):
                i = at[h]
                if not h:
                    rows[i] = -np.inf
                else:
                    t = h[1:]
                    while t not in at:
                        t = t[1:]
                    rows[i] = rows[at[t]] + self.backoff10.get(h, 0.0)
                for g in children.get(h, ()):
                    if g[-1] != LM_BOS:
                        rows[i, g[-1]] = self.logp10[g]
            self._tables["host"] = (keys[order], (rows * _LN10).astype(np.float32))
        return self._tables["host"]

    def device_arrays(self, device):
        """(keys (H,) int64 -- the uint64 keys' bits --, rows (H, K) float32) CUDA tensors on ``device``, uploaded on
        first use."""
        device = torch.device(device)
        if device not in self._tables:
            keys, rows = self.host_tables()
            self._tables[device] = (torch.from_numpy(keys.view(np.int64)).to(device), torch.from_numpy(rows).to(device))
        return self._tables[device]

    def descriptor(self, device):
        """The ``b2o_char_lm`` of this model on ``device`` (``_lib.CharLMDesc``)."""
        keys, rows = self.device_arrays(device)
        return _lib.CharLMDesc(self.order, keys.shape[0], keys.data_ptr(), rows.data_ptr(), self.alpha, self.beta)


class Hotwords:
    """Words to boost without requiring them, fused into the CTC prefix beam search (``b2o_crnn_forward_beam_hotword``;
    DESIGN.md section 1, "Hotwords").  A prefix is live when it is a prefix of a listed word (the empty prefix is).
    During the search a prefix a earns H(a) = ``weight`` * |a| while it is live and nothing once it leaves the list's
    trie; a returned reading keeps weight * |a| only if it is a listed word.  Readings rank by the acoustic score plus
    the language model's (if any) plus that bonus; the confidences stay acoustic.  Text outside the list reads as it
    does without hotwords, except where the bonus decides an ambiguous image.

    Entries are non-empty strings over ``alphabet`` of at most 48 characters, distinct, at most 2^20 of them and 2^24
    characters in all; the alphabet has at most 126 characters (the language-model kernel's class bound) and
    ``weight`` is a number >= 0, finite in float32.  Anything else raises ``ValueError`` naming the first offending entry
    or value.  An empty list is valid and changes nothing.

    The trie is compiled once on the host (``host_tables``) and uploaded lazily, once per CUDA device, so one object
    serves every rank of a sharded run.  A plain list or tuple of strings is accepted wherever a ``Hotwords`` is and is
    compiled for that call with the default weight."""

    WEIGHT = 1.5       # picked by scripts/bench_hotwords.py's sweep on its tuning pages (DESIGN.md section 5)

    def __init__(self, words, weight=WEIGHT, alphabet=DEFAULT_ALPHABET):
        if isinstance(words, str) or not isinstance(words, (list, tuple)):
            raise ValueError("hotwords are a list or tuple of strings")
        if len(alphabet) > _lib.MAX_LM_CLASSES - 1:
            raise ValueError(f"hotwords take an alphabet of at most {_lib.MAX_LM_CLASSES - 1} characters, "
                             f"got {len(alphabet)}")
        if len(words) > _lib.MAX_LEXICON_WORDS:
            raise ValueError(f"there are {len(words)} hotwords; at most {_lib.MAX_LEXICON_WORDS} are supported")
        index = {ch: i for i, ch in enumerate(alphabet)}
        seen = set()
        total = 0
        for i, w in enumerate(words):
            _check_word(i, w, index, "hotword")
            if w in seen:
                raise ValueError(f"hotword {i} ({w!r}) is a duplicate")
            seen.add(w)
            total += len(w)
            if total > _lib.MAX_LEXICON_LABELS:
                raise ValueError(f"hotword {i} ({w!r}) takes the list past {_lib.MAX_LEXICON_LABELS} characters in all")
        self._check_weight(weight)
        self.words, self.alphabet, self.weight = tuple(words), alphabet, float(weight)
        self._tables = {"host": compile_trie(self.words, index)}   # shared by weighted copies, with the uploads

    @staticmethod
    def _check_weight(weight):
        ok = not isinstance(weight, (bool, np.bool_)) and isinstance(weight, (int, float, np.integer, np.floating))
        if ok:
            with np.errstate(over="ignore"):
                ok = math.isfinite(float(np.float32(weight))) and float(weight) >= 0
        if not ok:
            raise ValueError(f"weight must be a number >= 0, finite in float32, got {weight!r}")

    def __len__(self):
        return len(self.words)

    def __repr__(self):
        return f"Hotwords({len(self.words)} words, weight={self.weight})"

    def weighted(self, weight=WEIGHT):
        """A copy with weight ``weight`` that shares this list's trie and device uploads."""
        self._check_weight(weight)
        other = object.__new__(Hotwords)
        other.__dict__.update(self.__dict__)
        other.weight = float(weight)
        return other

    def host_tables(self):
        """The trie (``compile_trie``): (keys (E,) uint64, child (E,) int32, final (N,) uint8), E = N - 1."""
        return self._tables["host"]

    def device_arrays(self, device):
        """(keys (E,) int64 -- the uint64 keys' bits --, child (E,) int32, final (N,) uint8) CUDA tensors on
        ``device``, uploaded on first use."""
        device = torch.device(device)
        if device not in self._tables:
            keys, child, final = self.host_tables()
            self._tables[device] = tuple(torch.from_numpy(a).to(device) for a in (keys.view(np.int64), child, final))
        return self._tables[device]

    def descriptor(self, device):
        """The ``b2o_hotwords`` of this list on ``device`` (``_lib.HotwordsDesc``)."""
        keys, child, final = self.device_arrays(device)
        ptr = lambda t: t.data_ptr() if t.numel() else None      # noqa: E731
        return _lib.HotwordsDesc(final.numel(), keys.numel(), ptr(keys), ptr(child), final.data_ptr(), self.weight)


def compile_trie(words, index):
    """The trie of checked, distinct ``words`` (``index``: character -> label), deterministic: nodes numbered
    breadth-first by (depth, parent, label), the root 0 the empty prefix.  Returns (keys (E,) uint64 ascending, key =
    (parent << 8) | label, child (E,) int32 the child of each edge -- so a node's children are contiguous --, final
    (N,) uint8, 1 where the node's prefix is a listed word), E = N - 1 edges."""
    nested = [{}]                                 # build ids -> {label: build id}
    ends = [False]
    for w in words:
        u = 0
        for ch in w:
            c = index[ch]
            v = nested[u].get(c)
            if v is None:
                v = nested[u][c] = len(nested)
                nested.append({})
                ends.append(False)
            u = v
        ends[u] = True
    n = len(nested)
    new = np.zeros(n, np.int64)                   # build id -> node
    parent = np.zeros(n, np.int64)                # node -> its parent and label
    label = np.zeros(n, np.int64)
    order = [0]                                   # build ids in node order; grows while it is walked
    for pos in range(n):
        u = order[pos]
        for c in sorted(nested[u]):
            v = nested[u][c]
            new[v], parent[len(order)], label[len(order)] = len(order), pos, c
            order.append(v)
    final = np.zeros(n, np.uint8)
    final[new[np.flatnonzero(np.asarray(ends))]] = 1
    # parents are non-decreasing in node order and a parent's children follow in label order: the keys ascend, and
    # the child of edge j is node j + 1
    keys = (parent[1:].astype(np.uint64) << np.uint64(8)) | label[1:].astype(np.uint64)
    return keys, np.arange(1, n, dtype=np.int32), final


class Pattern:
    """A regular expression every reading must match in full, enforced inside the CTC prefix beam search
    (``b2o_crnn_forward_beam_pattern``; DESIGN.md section 1, "Patterns"): a reading is returned only if
    ``re.fullmatch(regex, reading)`` accepts it.  The syntax is a strict subset of Python's ``re`` -- literals, ``\\``
    escapes of punctuation, ``.``, ``\\d``, classes with ranges and ``^``, groups, ``|`` and the quantifiers ``?``, ``*``,
    ``+``, ``{m}``, ``{m,}``, ``{m,n}`` with n <= 48 -- over ``alphabet``; everything else raises ``ValueError`` naming
    its position (``patterns``).  So do an automaton past 4096 states and a pattern whose shortest reading is longer
    than 48 characters.

    The pattern is compiled once on the host to its minimal trimmed DFA and uploaded lazily, once per CUDA device, so
    one object serves every rank of a sharded run.  A plain ``str`` is accepted wherever a ``Pattern`` is and is
    compiled for that call."""

    def __init__(self, regex, alphabet=DEFAULT_ALPHABET):
        from . import patterns
        self.regex, self.alphabet = regex, alphabet
        self.trans, self.dist, self.start = patterns.compile_pattern(regex, alphabet)
        self._index = {ch: i for i, ch in enumerate(alphabet)}
        self._device = {}

    @property
    def n_states(self):
        return int(self.trans.shape[0])

    def __repr__(self):
        return f"Pattern({self.regex!r}, {self.n_states} states)"

    def fullmatch(self, text):
        """Whether the DFA accepts ``text`` (a str), run on the host."""
        q = self.start
        for ch in text:
            c = self._index.get(ch)
            if c is None:
                return False
            q = int(self.trans[q, c])
            if q < 0:
                return False
        return bool(self.dist[q] == 0)

    def host_tables(self):
        """(trans (n, K-1) int16, -1 where there is no transition; dist (n,) uint8, the fewest labels to an accepting
        state, 0 for an accepting one, saturated at 255; start)."""
        return self.trans, self.dist, self.start

    def device_arrays(self, device):
        """(trans, dist) CUDA tensors on ``device``, uploaded on first use."""
        device = torch.device(device)
        if device not in self._device:
            self._device[device] = (torch.from_numpy(self.trans).to(device), torch.from_numpy(self.dist).to(device))
        return self._device[device]

    def descriptor(self, device):
        """The ``b2o_pattern`` of this pattern on ``device`` (``_lib.PatternDesc``)."""
        trans, dist = self.device_arrays(device)
        return _lib.PatternDesc(self.n_states, self.start, trans.data_ptr(), dist.data_ptr())


def check_hotwords(hotwords, beam_width=None, top_paths=1, lexicon=None, alphabet=DEFAULT_ALPHABET, pattern=None):
    """Validates a hotword choice before anything is launched (``ValueError`` otherwise) and returns the ``Hotwords`` to
    decode with, or None for ``hotwords=None``.  A ``Hotwords`` over ``alphabet`` or a list / tuple of strings
    (compiled here with the default weight) boosts its words in the beam search: it needs ``beam_width`` and does not
    combine with a lexicon or a pattern; it combines with a language model."""
    if hotwords is None:
        return None
    if not isinstance(hotwords, (Hotwords, list, tuple)):
        raise ValueError(f"hotwords must be a Hotwords or a list of strings, got {type(hotwords).__name__}")
    if beam_width is None:
        raise ValueError("hotwords need beam search: pass beam_width")
    if lexicon is not None:
        raise ValueError("lexicon and hotwords are mutually exclusive")
    if pattern is not None:
        raise ValueError("pattern and hotwords do not combine in one search")
    check_beam(beam_width, top_paths)
    if not isinstance(hotwords, Hotwords):
        return Hotwords(hotwords, alphabet=alphabet)
    if hotwords.alphabet != alphabet:
        raise ValueError("the hotwords were compiled for another alphabet than the recognizer's")
    return hotwords


def check_pattern(pattern, beam_width=None, top_paths=1, lexicon=None, alphabet=DEFAULT_ALPHABET, language_model=None,
                  hotwords=None):
    """Validates a pattern choice before anything is launched (``ValueError`` otherwise) and returns the ``Pattern`` to
    decode with, or None for ``pattern=None``.  A ``Pattern`` over ``alphabet`` or a ``str`` (compiled here) constrains
    the beam search: it needs ``beam_width`` and does not combine with a lexicon, a language model or hotwords."""
    if pattern is None:
        return None
    if not isinstance(pattern, (Pattern, str)):
        raise ValueError(f"pattern must be a Pattern or a str, got {type(pattern).__name__}")
    if beam_width is None:
        raise ValueError("a pattern needs beam search: pass beam_width")
    if lexicon is not None:
        raise ValueError("lexicon and pattern are mutually exclusive")
    if language_model is not None:
        raise ValueError("language_model and pattern do not combine in one search")
    if hotwords is not None:
        raise ValueError("pattern and hotwords do not combine in one search")
    check_beam(beam_width, top_paths)
    if isinstance(pattern, str):
        return Pattern(pattern, alphabet)
    if pattern.alphabet != alphabet:
        raise ValueError("the pattern was compiled for another alphabet than the recognizer's")
    return pattern


def check_decoder(beam_width=None, top_paths=1, lexicon=None, alphabet=DEFAULT_ALPHABET, language_model=None,
                  pattern=None, hotwords=None):
    """Validates a decoder choice before anything is launched (``ValueError`` otherwise) and returns the ``Lexicon`` to
    decode with, or None.  Without a lexicon this is ``check_beam``.  With one (a ``Lexicon`` over ``alphabet``, or a
    list / tuple of strings, compiled here): ``beam_width`` must be None and 1 <= ``top_paths`` <= 128.
    ``language_model`` (a ``CharLM`` over ``alphabet``) ranks the beam search by that model
    (``b2o_crnn_forward_beam_lm``): it needs ``beam_width`` and does not combine with a lexicon.
    ``pattern`` (a ``Pattern`` over ``alphabet`` or a str): the rules of ``check_pattern``, which returns the compiled
    pattern.  ``hotwords`` (a ``Hotwords`` over ``alphabet`` or a list of strings): the rules of ``check_hotwords``,
    which returns the compiled list; it combines with ``language_model``."""
    if pattern is not None:
        check_pattern(pattern, beam_width, top_paths, lexicon, alphabet, language_model, hotwords)
        return None
    if hotwords is not None:
        check_hotwords(hotwords, beam_width, top_paths, lexicon, alphabet)
        if language_model is None:
            return None
    if language_model is not None:
        if not isinstance(language_model, CharLM):
            raise ValueError(f"language_model must be a CharLM, got {type(language_model).__name__}")
        if lexicon is not None:
            raise ValueError("lexicon and language_model are mutually exclusive")
        if beam_width is None:
            raise ValueError("a language model needs beam search: pass beam_width")
        check_beam(beam_width, top_paths)
        if language_model.alphabet != alphabet:
            raise ValueError("the language model was built for another alphabet than the recognizer's")
        return None
    if lexicon is None:
        check_beam(beam_width, top_paths)
        return None
    if beam_width is not None:
        raise ValueError("lexicon and beam_width are mutually exclusive")
    if (not isinstance(top_paths, (int, np.integer)) or isinstance(top_paths, (bool, np.bool_))
            or not 1 <= top_paths <= _lib.MAX_LEXICON_TOP_PATHS):
        raise ValueError(f"with a lexicon, top_paths must be an int in [1, {_lib.MAX_LEXICON_TOP_PATHS}], got {top_paths!r}")
    if not isinstance(lexicon, Lexicon):
        lexicon = Lexicon(lexicon, alphabet)
    elif lexicon.alphabet != alphabet:
        raise ValueError("the lexicon was compiled for another alphabet than the recognizer's")
    return lexicon


ROTATION_VOTES = {"word": _lib.ROTATION_VOTE_WORD, "page": _lib.ROTATION_VOTE_PAGE}


def check_rotations(rotations=None, rotation_vote="word"):
    """Validates a choice of quarter turns before anything is launched (``ValueError`` otherwise) and returns the turns
    as a tuple of ints, or None.  ``rotations=None`` (the default) reads every crop as it is cut.  Otherwise a non-empty
    tuple or list of distinct ints from {0, 1, 2, 3}: every box is cut and decoded once per listed turn -- turn r starts
    the crop at corner r of the ordered box (tl, tr, br, bl), so a word on a page turned by ``np.rot90(page, k)`` reads
    upright in turn (4 - k) % 4 -- and ``rotation_vote`` picks one reading: ``"word"`` keeps, per word, the turn whose
    best reading has the largest log-probability; ``"page"`` keeps one turn per image, the one with the largest sum over
    the image's words.  Ties, and all -inf scores, go to the turn listed first."""
    if not isinstance(rotation_vote, str) or rotation_vote not in ROTATION_VOTES:
        raise ValueError(f"rotation_vote must be 'word' or 'page', got {rotation_vote!r}")
    if rotations is None:
        return None
    if not isinstance(rotations, (tuple, list)) or not rotations:
        raise ValueError(f"rotations must be None or a non-empty tuple or list of quarter turns, got {rotations!r}")
    for r in rotations:
        if not isinstance(r, (int, np.integer)) or isinstance(r, (bool, np.bool_)) or not 0 <= r <= 3:
            raise ValueError(f"rotations holds quarter turns 0, 1, 2 or 3, got {r!r}")
    turns = tuple(int(r) for r in rotations)
    if len(set(turns)) != len(turns):
        raise ValueError(f"rotations must be distinct, got {rotations!r}")
    return turns


def check_windows(max_windows=1, beam_width=None, lexicon=None, rotations=None, char_boxes=False, polygons=False,
                  char_scores=False):
    """Validates a choice of wide-word windows before anything is launched (``ValueError`` otherwise) and returns it as
    an int.  ``max_windows=1`` (the default) reads every box as one 200 x 31 crop, as warpBox cuts it.  An int 2 <= M <=
    16 reads every box wider than that crop at full height in up to M overlapping 200 x 31 windows and stitches their
    CTC steps into one reading (DESIGN.md section 1, "Wide words"); when a box of the call is wide the labels rows are
    48 M wide, -1 padded, and every other box reads exactly as with M = 1.  The windows are decoded greedily over 48
    steps each: with M > 1, ``beam_width``, ``lexicon``, ``rotations``, character boxes (``char_boxes``), polygons
    (``polygons``) and character scores (``char_scores``) raise: a stitched reading spans more than 48 steps."""
    if (not isinstance(max_windows, (int, np.integer)) or isinstance(max_windows, (bool, np.bool_))
            or not 1 <= max_windows <= _lib.MAX_WINDOWS):
        raise ValueError(f"max_windows must be an int in [1, {_lib.MAX_WINDOWS}], got {max_windows!r}")
    if max_windows > 1:
        excluded = [name for name, on in (("beam_width", beam_width is not None), ("lexicon", lexicon is not None),
                                          ("rotations", rotations is not None), ("return_char_boxes", char_boxes),
                                          ("return_polygons", polygons), ("return_char_scores", char_scores)) if on]
        if excluded:
            raise ValueError(f"max_windows > 1 reads wide words by greedy decoding only; it does not combine with "
                             f"{', '.join(excluded)}")
    return int(max_windows)


def check_char_scores(return_char_scores=False, char_alternatives=0):
    """Validates a request for character scores before anything is launched (``ValueError`` otherwise).  Returns None
    when ``return_char_scores`` is off, else A = ``char_alternatives``, an int in [0, 8]: every character of a reading
    gets its confidence and, with A > 0, the A most probable one-character edits at its position (``b2o_ctc_char_scores``,
    DESIGN.md section 1, "Character scores").  ``char_alternatives > 0`` without ``return_char_scores`` raises."""
    a = char_alternatives
    if (not isinstance(a, (int, np.integer)) or isinstance(a, (bool, np.bool_))
            or not 0 <= a <= _lib.MAX_CHAR_ALTERNATIVES):
        raise ValueError(f"char_alternatives must be an int in [0, {_lib.MAX_CHAR_ALTERNATIVES}], got {a!r}")
    if not return_char_scores:
        if a:
            raise ValueError("char_alternatives needs return_char_scores=True")
        return None
    return int(a)


def check_polygons(entries):
    """Validates the words of a box group on the host, before anything is launched, and returns them as the dense table
    ``b2o_warp_polys`` reads: (polys (B,18,2) float32, points (B,) int32), unused points NaN.  An entry is a (2m,2)
    array: a box (m = 2, four corners) or a polygon of m - 1 segments, 3 <= m <= 9 -- the top edge t_0 .. t_{m-1}
    left to right, then the bottom edge b_{m-1} .. b_0, as ``Detector.detect(return_polygons=True)`` returns them.
    ``ValueError`` names the first entry with an odd point count, too few or too many points, a non-finite value, or
    a degenerate segment (a quad t_i, t_i+1, b_i+1, b_i with coinciding corners or zero area)."""
    n = len(entries)
    polys = np.full((n, _lib.POLY_POINTS, 2), np.nan, np.float32)
    points = np.zeros(n, np.int32)
    for i, e in enumerate(entries):
        a = np.asarray(e, dtype=np.float32)
        if a.ndim != 2 or a.shape[1] != 2:
            raise ValueError(f"entry {i} has shape {a.shape}: a word is a (points, 2) array")
        p = a.shape[0]
        if p % 2:
            raise ValueError(f"entry {i} has an odd number of points ({p})")
        if p < 4 or p > _lib.POLY_POINTS:
            raise ValueError(f"entry {i} has {p} points: a word has 4 (a box) or 6 to {_lib.POLY_POINTS} (a polygon)")
        if not np.isfinite(a).all():
            raise ValueError(f"entry {i} has a non-finite coordinate")
        if p > 4:
            s = p // 2 - 1
            for j in range(s):
                q = a[[j, j + 1, p - 2 - j, p - 1 - j]].astype(np.float64)
                x, y = q[:, 0], q[:, 1]
                area = 0.5 * (np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))
                same = (np.abs(q[:, None] - q[None]).max(-1) == 0).sum() > 4
                if same or area == 0:
                    raise ValueError(f"entry {i} has a degenerate segment {j}")
        polys[i, :p] = a
        points[i] = p
    return polys, points


def decode_paths(labels, alphabet=DEFAULT_ALPHABET, logp=None):
    """Host labels -> texts, and logp -> confidences (None without logp).  (B,48) labels / (B,) logp give B strings and
    a float32 array, as the greedy decoder returns them; (B,P,48) / (B,P) -- ``top_paths = P > 1`` -- give B lists of P
    strings and B lists of P confidences, best first."""
    labels = np.asarray(labels)
    if labels.ndim == 2:
        return labels_to_text(labels, alphabet), (None if logp is None else confidences(logp))
    b, p = labels.shape[:2]
    flat = labels_to_text(labels.reshape(b * p, STEPS), alphabet)
    texts = [flat[i * p:(i + 1) * p] for i in range(b)]
    return texts, (None if logp is None else [list(row) for row in confidences(logp)])


def char_boxes_host(cells, texts):
    """Host cells (B,48,4,2) or (B,P,48,4,2) float32 (``b2o_char_cells``) -> one (n,4,2) float32 array per word, n =
    len(text); with ``top_paths = P > 1`` (texts are lists of P strings) a list of P arrays per word."""
    cells = np.asarray(cells)
    if cells.ndim == 4:
        return [cells[i, :len(t)] for i, t in enumerate(texts)]
    return [[cells[i, j, :len(t)] for j, t in enumerate(row)] for i, row in enumerate(texts)]


def char_scores_host(conf, texts, alphabet=DEFAULT_ALPHABET, alt_labels=None, alt_post=None):
    """Host character scores (``b2o_ctc_char_scores``) -> one entry per word, n = len(text): conf (B,48) or (B,P,48)
    float32 gives an (n,) float32 array of the characters' confidences; with alt_labels / alt_post (B[,P],48,A) the
    entry is (that array, n lists of A (character, posterior) pairs, best first), the character ``''`` for the deletion
    and None for a slot without an edit (posterior 0).  With ``top_paths = P > 1`` (texts are lists of P strings) a list
    of P entries per word."""
    conf = np.asarray(conf)
    chars = list(alphabet) + [""]                                  # label K-1: the deletion

    def one(c, text, lab, post):
        n = len(text)
        if lab is None:
            return c[:n]
        alts = [[(chars[e] if e >= 0 else None, q) for e, q in zip(le, pe)]
                for le, pe in zip(lab[:n].tolist(), post[:n].tolist())]
        return c[:n], alts

    pick = (lambda a, *i: None if a is None else a[i])             # noqa: E731
    if conf.ndim == 2:
        return [one(conf[i], t, pick(alt_labels, i), pick(alt_post, i)) for i, t in enumerate(texts)]
    return [[one(conf[i, j], t, pick(alt_labels, i, j), pick(alt_post, i, j)) for j, t in enumerate(row)]
            for i, row in enumerate(texts)]


class Recognizer:
    """A text recognizer using the CRNN architecture, running as sm_90a CUDA kernels.

    Args:
        alphabet: the characters the model recognises (default ``0-9a-z``; up to 1023 characters).  The
            checkpoint's ``fc_12`` must have ``len(alphabet) + 1`` classes; if it does not, the reference's
            "backbone weights only" behaviour applies (recognition.py:399-411): the top layer is
            re-initialised (Glorot uniform, zero bias) and has to be trained before it is useful: ``fit_top`` trains it
            on the GPU from labelled word crops, and ``save_weights`` keeps the result.
        weights: ``None`` builds an untrained model for ``alphabet`` (as the reference does); ``"kurapan"`` looks for ``crnn_kurapan.npz`` (exported) or the reference's ``crnn_kurapan.h5``
            (read with h5py where installed) in the cache dir; otherwise a ``.npz`` / ``.h5`` path or a dict
            keyed like ``weights.py``.
        build_params: ``None`` / the defaults (reference recognition.py:13-23), optionally with ``"stn": False`` (the
            recognizer without the spatial transformer, recognition.py:243) and / or ``"color": True`` (RGB crops into a
            3-channel ``conv_1``, recognition.py:214); other architectures raise NotImplementedError.
    """

    def __init__(self, alphabet=None, weights="kurapan", build_params=None, device=None):
        assert alphabet or weights, "At least one of alphabet or weights must be provided."
        # build_params (recognition.py:13-23, 365-368): the CUDA recognizer implements the default architecture; of the
        # build options only ``stn`` (with / without the spatial transformer, recognition.py:243) and ``color`` (RGB instead
        # of gray crops, recognition.py:214) may differ
        params = dict(DEFAULT_BUILD_PARAMS, **(build_params or {}))
        self.stn = bool(params.pop("stn", True))
        self.color = bool(params["color"])                        # RGB crops, no gray conversion (recognition.py:214, 508-510)
        params["color"] = False
        if params != DEFAULT_BUILD_PARAMS:
            changed = sorted(k for k in params if params[k] != DEFAULT_BUILD_PARAMS.get(k))
            raise NotImplementedError(f"build_params other than the defaults are not supported by the CUDA recognizer: {changed}")
        if not torch.cuda.is_available():
            raise _lib.B2OError("keras-ocr_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.alphabet = alphabet or DEFAULT_ALPHABET              # recognition.py:369-375
        if len(self.alphabet) + 1 > _lib.MAX_CLASSES:
            raise ValueError(f"alphabet too long: at most {_lib.MAX_CLASSES - 1} characters")
        self.blank_label_idx = len(self.alphabet)
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        if isinstance(weights, dict):
            tensors = weights
        elif weights is None:
            # reference recognition.py:382-383: no weights -> the freshly built (untrained) model for this alphabet
            tensors = weights_mod.synthetic_crnn_weights(seed=0, alphabet=self.alphabet, stn=self.stn, color=self.color)
        elif isinstance(weights, str) and weights.endswith(".npz"):
            tensors = weights_mod.load_npz(weights)
        elif isinstance(weights, str) and weights.endswith(".h5"):
            tensors = weights_mod.load_keras_h5(weights)
        elif weights == "kurapan":                                # recognition.py:27-44: cache file, sha256-verified
            import os
            cache = tools.get_default_cache_dir()
            if os.path.isfile(os.path.join(cache, "crnn_kurapan.npz")):
                tensors = weights_mod.load_npz(os.path.join(cache, "crnn_kurapan.npz"))
            else:
                tensors = weights_mod.load_keras_h5(tools.find_cached(
                    "crnn_kurapan.h5", sha256="a7d8086ac8f5c3d6a0a828f7d6fbabcaf815415dd125c32533013f85603be46d"))
        else:
            raise NotImplementedError(f"Cannot load weights from {weights}")
        has_stn = "stn.conv_a.kernel" in tensors
        if has_stn and not self.stn:                              # stn=False with a checkpoint that has one: drop it
            tensors = {k: v for k, v in tensors.items() if not k.startswith("stn.")}
        elif self.stn and not has_stn:
            raise ValueError("the checkpoint has no spatial-transformer tensors: pass build_params={'stn': False}")
        in_ch = int(np.shape(tensors["conv_1.kernel"])[2]) if "conv_1.kernel" in tensors else 1
        if in_ch != (3 if self.color else 1):
            raise ValueError(f"conv_1.kernel takes {in_ch} input channel(s): pass build_params={{'color': {in_ch == 3}}}")
        n_classes = len(self.alphabet) + 1
        top = tensors.get("fc_12.kernel")
        if top is None or tuple(np.shape(top)) != (256, n_classes):
            print("Provided alphabet does not match pretrained alphabet. Using backbone weights only.")
            tensors = dict(tensors)
            limit = float(np.sqrt(6.0 / (256 + n_classes)))           # keras Dense default: glorot_uniform, zeros
            tensors["fc_12.kernel"] = np.random.default_rng(0).uniform(-limit, limit, (256, n_classes)).astype(np.float32)
            tensors["fc_12.bias"] = np.zeros(n_classes, np.float32)
        self.ctx = _lib.Context(self.device_index)
        self.ctx.load_crnn(tensors)
        self._tensors = tensors          # host weights as loaded (save_weights; fit_top replaces the top)
        self._keep_workspace = False     # tests set keep_workspace to read intermediate taps
        self._last_ws = None
        self._ws = None                  # reusable CRNN workspace (grown on demand)

    @property
    def keep_workspace(self):
        return self._keep_workspace

    @keep_workspace.setter
    def keep_workspace(self, on):
        """Debug: keep the last forward pass's workspace for ``tap`` and make the CRNN write its fp32 logits
        (off on the product path: the fused Dense + CTC kernel then stores labels only)."""
        self._keep_workspace = bool(on)
        self.ctx.set_debug_taps(self._keep_workspace)

    # ------------------------------------------------------------------ device-resident API
    def gray_device(self, images_t):
        n, h, w, _ = images_t.shape
        gray = torch.empty((n, h, w), dtype=torch.uint8, device=self.device)
        self.ctx.rgb_to_gray(images_t.data_ptr(), n, h, w, gray.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
        return gray

    def warp_device(self, gray, boxes_flat, image_index, want_crops=False, turn=None):
        """tools.warpBox for every box.  ``gray``: (N,H,W) u8 -- or the RGB batch (N,H,W,3) for a color recognizer.
        ``turn`` (0..3): the crops in that quarter turn (``b2o_warp_boxes_turned``, see ``check_rotations``).
        Returns (crnn_in (B,200,31[,3]) fp16, crops (B,31,200[,3]) u8 or None)."""
        n, h, w = gray.shape[:3]
        color = gray.dim() == 4
        assert color == self.color, "a color recognizer warps the RGB batch, a gray one the gray batch"
        tail = (3,) if color else ()
        b = boxes_flat.shape[0]
        crnn_in = torch.empty((b, TARGET_WIDTH, TARGET_HEIGHT) + tail, dtype=torch.float16, device=self.device)
        crops = torch.empty((b, TARGET_HEIGHT, TARGET_WIDTH) + tail, dtype=torch.uint8, device=self.device) if want_crops else None
        stream = torch.cuda.current_stream(self.device).cuda_stream
        if turn is None:
            self.ctx.warp_boxes(gray.data_ptr(), n, h, w, boxes_flat.data_ptr(), image_index.data_ptr(), b,
                                crops.data_ptr() if want_crops else None, crnn_in.data_ptr(), stream, color=color)
        else:
            self.ctx.warp_boxes_turned(gray.data_ptr(), 3 if color else 1, n, h, w, boxes_flat.data_ptr(),
                                       image_index.data_ptr(), b, int(turn), crops.data_ptr() if want_crops else None,
                                       crnn_in.data_ptr(), stream)
        return crnn_in, crops

    def warp_polys_device(self, gray, polys, points, image_index, want_crops=False):
        """warpBox along every polygon (``b2o_warp_polys``): polys (B,18,2) float32 and points (B,) int32 CUDA as
        ``check_polygons`` / ``b2o_compact_polys`` lay them out; a 4-point entry is cut as ``warp_device`` cuts it.
        Returns (crnn_in, crops or None) as ``warp_device`` does."""
        n, h, w = gray.shape[:3]
        color = gray.dim() == 4
        assert color == self.color, "a color recognizer warps the RGB batch, a gray one the gray batch"
        tail = (3,) if color else ()
        b = polys.shape[0]
        crnn_in = torch.empty((b, TARGET_WIDTH, TARGET_HEIGHT) + tail, dtype=torch.float16, device=self.device)
        crops = torch.empty((b, TARGET_HEIGHT, TARGET_WIDTH) + tail, dtype=torch.uint8, device=self.device) if want_crops else None
        self.ctx.warp_polys(gray.data_ptr(), 3 if color else 1, n, h, w, polys.data_ptr(), points.data_ptr(),
                            image_index.data_ptr(), b, crops.data_ptr() if want_crops else None, crnn_in.data_ptr(),
                            torch.cuda.current_stream(self.device).cuda_stream)
        return crnn_in, crops

    def window_counts_device(self, flat, max_windows):
        """``b2o_window_counts`` of a dense box list: flat (B,4,2) float32 CUDA -> K (B,) int32 CUDA, the windows every
        box is read in with ``max_windows`` (1 for a box that fits the 200 x 31 crop at full height)."""
        b = flat.shape[0]
        out = torch.empty((b,), dtype=torch.int32, device=self.device)
        self.ctx.window_counts(flat.data_ptr(), None, 1, b, int(max_windows), out.data_ptr(),
                               torch.cuda.current_stream(self.device).cuda_stream)
        return out

    def _read_windowed(self, gray, flat, image_index, max_windows, windows, with_scores):
        """Warp + CRNN + greedy CTC of every box, then every wide box (K >= 2 in ``windows``, host ints (B,), or None:
        computed here and read back) read again in its K windows and stitched: (labels, logp (B,) or None) CUDA, labels
        (B,48 M) int32 -1 padded, or the default read's (B,48) when no box is wide.  The windows go through the CRNN in
        chunks of at most B crops, so the CRNN workspace stays that of the default read; only their logits and theta are
        kept for ``b2o_stitch_windows``.  With ``windows`` given nothing here waits for the device: the word list and the
        CSR of window starts travel through pinned memory."""
        b, m = flat.shape[0], int(max_windows)
        if windows is None:
            windows = self.window_counts_device(flat, m).cpu().numpy()
        windows = np.asarray(windows)
        crnn_in, _ = self.warp_device(gray, flat, image_index)
        read = self.predict_device(crnn_in, with_scores=with_scores)
        labels, logp = read if with_scores else (read, None)
        del crnn_in
        wide = np.flatnonzero(windows >= 2)
        if wide.size == 0:
            return labels, logp
        out = torch.full((b, STEPS * m), -1, dtype=torch.int32, device=self.device)
        out[:, :STEPS] = labels
        csr = torch.empty((2 * wide.size + 1,), dtype=torch.int32, pin_memory=True)     # words, then window starts
        host = csr.numpy()
        host[:wide.size] = wide
        host[wide.size] = 0
        host[wide.size + 1:] = np.cumsum(windows[wide])
        csr_t = csr.to(self.device, non_blocking=True)  # the pinned block is not reused before this copy has run
        words_t, start_t = csr_t[:wide.size], csr_t[wide.size:]
        total, k = int(host[-1]), len(self.alphabet) + 1
        logits = torch.empty((total, STEPS, k), dtype=torch.float32, device=self.device)
        theta = torch.empty((total, 6), dtype=torch.float32, device=self.device) if self.stn else None
        chunk = min(b, total)
        tail = (3,) if self.color else ()
        x = torch.empty((chunk, TARGET_WIDTH, TARGET_HEIGHT) + tail, dtype=torch.float16, device=self.device)
        greedy = torch.empty((chunk, STEPS), dtype=torch.int32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        n, h, w = gray.shape[:3]
        for first in range(0, total, chunk):
            c = min(chunk, total - first)
            self.ctx.warp_windows(gray.data_ptr(), 3 if self.color else 1, n, h, w, flat.data_ptr(),
                                  image_index.data_ptr(), words_t.data_ptr(), start_t.data_ptr(), wide.size, m, first, c,
                                  None, x.data_ptr(), stream)
            nbytes = self.ctx.crnn_workspace_bytes(c)
            if self._ws is None or self._ws.numel() < nbytes:
                self._ws = None
                self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            ws = self._ws.data_ptr()
            self.ctx.crnn_forward_logits(x.data_ptr(), c, greedy.data_ptr(), None, ws, nbytes, stream)
            self.ctx.crnn_tap("logits", ws, c, logits[first].data_ptr(), c * STEPS * k * 4, stream)
            if theta is not None:
                self.ctx.crnn_tap("theta", ws, c, theta[first].data_ptr(), c * 6 * 4, stream)
        self.ctx.stitch_windows(logits.data_ptr(), k, None if theta is None else theta.data_ptr(), flat.data_ptr(),
                                words_t.data_ptr(), start_t.data_ptr(), wide.size, m, out.data_ptr(),
                                None if logp is None else logp.data_ptr(), stream)
        return out, logp

    def _decoder(self, beam_width, top_paths, lexicon, language_model=None, pattern=None, hotwords=None):
        """``check_decoder`` for this recognizer's alphabet: (the compiled lexicon or None, the compiled pattern or
        None, the compiled hotwords or None)."""
        if pattern is not None:
            return None, check_pattern(pattern, beam_width, top_paths, lexicon, self.alphabet, language_model,
                                       hotwords), None
        if hotwords is not None:
            hotwords = check_hotwords(hotwords, beam_width, top_paths, lexicon, self.alphabet)
            check_decoder(beam_width, top_paths, None, self.alphabet, language_model)
            return None, None, hotwords
        plain = lexicon is None and language_model is None
        return check_decoder(beam_width, top_paths, lexicon, DEFAULT_ALPHABET if plain else self.alphabet,
                             language_model), None, None

    def predict_device(self, crnn_in, with_scores=False, beam_width=None, top_paths=1, lexicon=None,
                       language_model=None, pattern=None, char_scores=None, hotwords=None):
        """CRNN + greedy CTC.  crnn_in: (B,200,31) fp16 -> labels (B,48) int32 (-1 padded).  ``with_scores``: returns
        (labels, logp) with logp (B,) float32 the greedy path's log-probability (``b2o_crnn_forward_scored``).
        ``beam_width``: CTC prefix beam search instead (``b2o_crnn_forward_beam``, see ``check_beam``), logp = the beam
        scores; ``top_paths > 1`` gives labels (B,P,48) and logp (B,P), best first.  ``lexicon`` (a ``Lexicon`` or a
        list of strings, see ``check_decoder``): the ``top_paths`` most probable entries instead
        (``b2o_crnn_forward_lexicon``), logp = their CTC forward log-probabilities, in the same shapes.
        ``language_model`` (a ``CharLM``, with ``beam_width``): the beam search ranked by that model
        (``b2o_crnn_forward_beam_lm``); logp stays the acoustic beam score of each reading.  ``pattern`` (a
        ``Pattern`` or a str, with ``beam_width``): only readings that match it in full (``b2o_crnn_forward_beam_pattern``),
        logp their beam scores; slots past a crop's matching readings are -1 with logp -inf.  ``hotwords`` (a
        ``Hotwords`` or a list of strings, with ``beam_width``, with or without ``language_model``): the beam search
        with a bonus for the listed words (``b2o_crnn_forward_beam_hotword``); logp stays the acoustic beam score.
        ``char_scores`` = A (``check_char_scores``): the result also ends with every reading's character confidences
        (B,48) float32 and, with A > 0, its alternatives' labels (B,48,A) int32 and posteriors (B,48,A) float32
        (``b2o_crnn_char_scores``); (B,P,48) / (B,P,48,A) with ``top_paths = P > 1``."""
        lexicon, pattern, hotwords = self._decoder(beam_width, top_paths, lexicon, language_model, pattern, hotwords)
        b = crnn_in.shape[0]
        lead = (b,) if top_paths == 1 else (b, top_paths)
        labels = torch.empty(lead + (STEPS,), dtype=torch.int32, device=self.device)
        logp = torch.empty(lead, dtype=torch.float32, device=self.device) if with_scores else None
        scores = None if char_scores is None else self._score_buffers(lead, char_scores)
        self._forward(crnn_in, labels, logp, beam_width, top_paths, lexicon, language_model=language_model,
                      pattern=pattern, char_scores=scores, hotwords=hotwords)
        if scores is not None:
            return ((labels, logp) if with_scores else (labels,)) + tuple(t for t in scores if t is not None)
        return (labels, logp) if with_scores else labels

    def _score_buffers(self, lead, alternatives):
        """Device outputs of ``b2o_crnn_char_scores`` for readings of shape ``lead``: (conf, alternative labels,
        posteriors), the last two None when ``alternatives`` is 0."""
        conf = torch.empty(lead + (STEPS,), dtype=torch.float32, device=self.device)
        if not alternatives:
            return conf, None, None
        return (conf, torch.empty(lead + (STEPS, alternatives), dtype=torch.int32, device=self.device),
                torch.empty(lead + (STEPS, alternatives), dtype=torch.float32, device=self.device))

    def _forward(self, crnn_in, labels, logp, beam_width, top_paths, lexicon, spans=None, theta=None,
                 language_model=None, fused=None, pattern=None, char_scores=None, hotwords=None):
        """The CRNN and the decoder of ``predict_device`` into caller-allocated ``labels`` / ``logp`` (None: greedy
        without scores, or scores not written); ``lexicon`` is already compiled.  With ``language_model``, ``fused``
        (B,P) float32 or None receives every reading's F_end, and so it does with ``hotwords`` (already compiled).
        ``pattern`` is already compiled.  ``spans`` (B,P,48,2) int32: also the
        characters' emission spans of every reading (``b2o_crnn_align``) and, with an STN, its ``theta`` (B,6) float32;
        the greedy forward then keeps its logits (``b2o_crnn_forward_logits``).  ``char_scores``: (conf, alternative
        labels or None, posteriors or None) of ``_score_buffers``, filled by ``b2o_crnn_char_scores`` after the decoder
        (the greedy forward then keeps its logits too)."""
        b = crnn_in.shape[0]
        nbytes = self.ctx.crnn_workspace_bytes(b)
        if lexicon is not None:
            nbytes = (nbytes + 255) // 256 * 256 + self.ctx.lexicon_workspace_bytes(b, len(lexicon), int(top_paths))
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        ws = self._ws
        stream = torch.cuda.current_stream(self.device).cuda_stream
        logp_ptr = logp.data_ptr() if logp is not None else None
        if lexicon is not None:
            offsets, lex_labels = lexicon.device_arrays(self.device)
            self.ctx.crnn_forward_lexicon(crnn_in.data_ptr(), b, offsets.data_ptr(), lex_labels.data_ptr(), len(lexicon),
                                          int(top_paths), labels.data_ptr(), logp_ptr, ws.data_ptr(), nbytes, stream)
        elif hotwords is not None:
            self.ctx.crnn_forward_beam_hotword(crnn_in.data_ptr(), b, int(beam_width), int(top_paths),
                                               None if language_model is None else language_model.descriptor(self.device),
                                               hotwords.descriptor(self.device), labels.data_ptr(), logp_ptr,
                                               fused.data_ptr() if fused is not None else None, ws.data_ptr(), nbytes,
                                               stream)
        elif language_model is not None:
            self.ctx.crnn_forward_beam_lm(crnn_in.data_ptr(), b, int(beam_width), int(top_paths),
                                          language_model.descriptor(self.device), labels.data_ptr(), logp_ptr,
                                          fused.data_ptr() if fused is not None else None, ws.data_ptr(), nbytes,
                                          stream)
        elif pattern is not None:
            self.ctx.crnn_forward_beam_pattern(crnn_in.data_ptr(), b, int(beam_width), int(top_paths),
                                               pattern.descriptor(self.device), labels.data_ptr(), logp_ptr,
                                               ws.data_ptr(), nbytes, stream)
        elif beam_width is not None:
            self.ctx.crnn_forward_beam(crnn_in.data_ptr(), b, int(beam_width), int(top_paths), labels.data_ptr(),
                                       logp_ptr, ws.data_ptr(), nbytes, stream)
        elif spans is not None or char_scores is not None:
            self.ctx.crnn_forward_logits(crnn_in.data_ptr(), b, labels.data_ptr(), logp_ptr, ws.data_ptr(), nbytes,
                                         stream)
        elif logp is not None:
            self.ctx.crnn_forward_scored(crnn_in.data_ptr(), b, labels.data_ptr(), logp_ptr, ws.data_ptr(), nbytes,
                                         stream)
        else:
            self.ctx.crnn_forward(crnn_in.data_ptr(), b, labels.data_ptr(), ws.data_ptr(), nbytes, stream)
        if spans is not None:
            self.ctx.crnn_align(b, labels.data_ptr(), int(top_paths), spans.data_ptr(), None,
                                theta.data_ptr() if theta is not None else None, ws.data_ptr(), nbytes, stream)
        if char_scores is not None:
            conf, alt_labels, alt_post = char_scores
            ptr = lambda t: t.data_ptr() if t is not None else None      # noqa: E731
            self.ctx.crnn_char_scores(b, labels.data_ptr(), int(top_paths), 0 if alt_labels is None else alt_labels.shape[-1],
                                      conf.data_ptr(), ptr(alt_labels), ptr(alt_post), None, ws.data_ptr(), nbytes, stream)
        self._last_ws = (ws, b) if self.keep_workspace else None

    def _predict_aligned(self, crnn_in, beam_width, top_paths, lexicon, language_model=None, pattern=None,
                         char_scores=None, hotwords=None):
        """``predict_device(with_scores=True)`` plus every reading's spans: (labels (B,P,48), logp (B,P), spans
        (B,P,48,2) int32, theta (B,6) float32 or None without an STN), followed by the ``_score_buffers`` of
        ``char_scores`` = A when it is given."""
        b, p = crnn_in.shape[0], int(top_paths)
        labels = torch.empty((b, p, STEPS), dtype=torch.int32, device=self.device)
        logp = torch.empty((b, p), dtype=torch.float32, device=self.device)
        spans = torch.empty((b, p, STEPS, 2), dtype=torch.int32, device=self.device)
        theta = torch.empty((b, 6), dtype=torch.float32, device=self.device) if self.stn else None
        scores = None if char_scores is None else self._score_buffers((b, p), char_scores)
        self._forward(crnn_in, labels, logp, beam_width, p, lexicon, spans, theta, language_model, pattern=pattern,
                      char_scores=scores, hotwords=hotwords)
        return (labels, logp, spans, theta) + (() if scores is None else (scores,))

    def char_cells_device(self, spans, theta, boxes=None, turns=None):
        """``b2o_char_cells``: spans (B,P,48,2) int32, theta (B,6) or None, boxes (B,4,2) float32 as they were cut (None:
        the 200 x 31 crop frame), turns (B,) int32 or None -> cells (B,P,48,4,2) float32 CUDA."""
        b, p = spans.shape[:2]
        cells = torch.empty((b, p, STEPS, 4, 2), dtype=torch.float32, device=self.device)
        ptr = lambda t: t.data_ptr() if t is not None else None      # noqa: E731
        self.ctx.char_cells(spans.data_ptr(), b, p, ptr(theta), ptr(boxes), ptr(turns), cells.data_ptr(),
                            torch.cuda.current_stream(self.device).cuda_stream)
        return cells

    def tap(self, name, shape, dtype):
        """Debug: copy an intermediate of the last predict_device call (needs keep_workspace=True)."""
        ws, b = self._last_ws
        out = torch.empty(shape, dtype=dtype, device=self.device)
        self.ctx.crnn_tap(name, ws.data_ptr(), b, out.data_ptr(), out.numel() * out.element_size(),
                          torch.cuda.current_stream(self.device).cuda_stream)
        return out

    def recognize_crops(self, crops, return_scores=False, beam_width=None, top_paths=1, lexicon=None,
                        return_char_boxes=False, language_model=None, pattern=None, return_char_scores=False,
                        char_alternatives=0, hotwords=None):
        """crops: (B,31,200) uint8 -- (B,31,200,3) for a color recognizer -- i.e. what tools.warpBox returns -> list[str].
        ``return_scores=True``: a list of (text, confidence) instead, see ``confidences``.  ``beam_width``: beam search
        decoding (``check_beam``); with ``top_paths = P > 1`` each text is a list of P strings and each confidence a
        list of P floats, best first (``decode_paths``).  ``lexicon``: the most probable entries of a word list instead
        (``check_decoder``), in the same shapes; a confidence is exp(the entry's CTC log-probability), clipped to 1.
        ``language_model`` (a ``CharLM``, with ``beam_width``): the beam search ranked by that character model; the
        confidences stay exp(the acoustic beam score).  ``pattern`` (a ``Pattern`` or a str, with ``beam_width``): only
        readings that match it in full; a word with no matching reading reads "" with confidence 0.  ``hotwords`` (a
        ``Hotwords`` or a list of strings, with ``beam_width``, alone or with ``language_model``): listed words win
        where the image is ambiguous, everything else reads as without them; the confidences stay acoustic.
        ``return_char_boxes=True``: every word is a tuple that ends with its character cells (``b2o_char_cells``), an
        (n,4,2) float32 array for a text of n characters (a list of P arrays with ``top_paths = P > 1``), in the crop's
        200 x 31 frame: (text, cells) or (text, confidence, cells).
        ``return_char_scores=True``: every word's tuple ends with its character scores (``check_char_scores``,
        ``char_scores_host``), after the cells when both are asked for: an (n,) float32 array of the characters'
        confidences, or with ``char_alternatives = A > 0`` that array and n lists of A (character, posterior) pairs;
        a list of P of these with ``top_paths = P > 1``.  They are acoustic: they do not depend on the decoder."""
        lexicon, pattern, hotwords = self._decoder(beam_width, top_paths, lexicon, language_model, pattern, hotwords)
        char_scores = check_char_scores(return_char_scores, char_alternatives)
        t = crops if isinstance(crops, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(crops))
        t = t.to(self.device).contiguous()
        b = t.shape[0]
        if b == 0:
            return []
        assert t.shape[1:] == (TARGET_HEIGHT, TARGET_WIDTH) + ((3,) if self.color else ()), "crops must be (B,31,200[,3])"
        crnn_in = torch.empty((b, TARGET_WIDTH, TARGET_HEIGHT) + ((3,) if self.color else ()), dtype=torch.float16, device=self.device)
        self.ctx.crops_to_input(t.data_ptr(), b, crnn_in.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream,
                                color=self.color)
        beam = {"beam_width": beam_width, "top_paths": top_paths, "lexicon": lexicon, "language_model": language_model,
                "pattern": pattern, "hotwords": hotwords}
        if return_char_boxes:
            labels, logp, spans, theta, *scores = self._predict_aligned(crnn_in, char_scores=char_scores, **beam)
            return self._host_words(labels, logp, top_paths, return_scores, self.char_cells_device(spans, theta),
                                    scores[0] if scores else None)
        if char_scores is not None:
            labels, logp, *scores = self.predict_device(crnn_in, with_scores=True, char_scores=char_scores, **beam)
            return self._host_words(labels, logp, top_paths, return_scores, None, scores)
        if not return_scores:
            return decode_paths(self.predict_device(crnn_in, **beam).cpu().numpy(), self.alphabet)[0]
        labels, logp = self.predict_device(crnn_in, with_scores=True, **beam)
        return list(zip(*decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())))

    def _host_words(self, labels, logp, top_paths, return_scores, cells=None, scores=None):
        """Host words of ``recognize_crops`` / ``recognize_from_boxes`` with cells and / or character scores:
        (text[, confidence][, cells][, character scores]).  ``scores``: the device tensors of ``_score_buffers``
        (None entries are skipped), or None."""
        scores = None if scores is None else [t for t in scores if t is not None]
        if top_paths == 1 and labels.dim() == 3:
            labels, logp = labels[:, 0], logp[:, 0]
            cells = None if cells is None else cells[:, 0]
            scores = None if scores is None else [t[:, 0] for t in scores]
        texts, conf = decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())
        cols = [texts] + ([conf] if return_scores else [])
        if cells is not None:
            cols.append(char_boxes_host(cells.cpu().numpy(), texts))
        if scores is not None:
            host = [t.cpu().numpy() for t in scores]
            cols.append(char_scores_host(host[0], texts, self.alphabet, *host[1:]))
        return list(zip(*cols))

    def recognize(self, image, beam_width=None, top_paths=1, lexicon=None, language_model=None, pattern=None,
                  hotwords=None):
        """Recognize text from a single pre-cropped image (reference recognition.py:467-489): fit to
        200x31 with zero fill (host, as upstream), gray conversion, then the CUDA CRNN.  ``beam_width`` / ``top_paths`` /
        ``lexicon`` / ``language_model`` / ``pattern`` / ``hotwords``: as ``recognize_crops``."""
        import cv2

        lexicon, pattern, hotwords = self._decoder(beam_width, top_paths, lexicon, language_model, pattern, hotwords)
        image = tools.read_and_fit(filepath_or_array=image, width=TARGET_WIDTH, height=TARGET_HEIGHT, cval=0)
        if not self.color and image.ndim == 3 and image.shape[-1] == 3:      # recognition.py:481-483
            image = cv2.cvtColor(image, code=cv2.COLOR_RGB2GRAY)
        return self.recognize_crops(np.ascontiguousarray(image.reshape((1, TARGET_HEIGHT, TARGET_WIDTH) + ((3,) if self.color else ()))),
                                    beam_width=beam_width, top_paths=top_paths, lexicon=lexicon,
                                    language_model=language_model, pattern=pattern, hotwords=hotwords)[0]

    def recognize_from_boxes_device(self, images_t, boxes, counts, gray=None, flat=None, image_index=None,
                                    with_scores=False, beam_width=None, top_paths=1, lexicon=None, rotations=None,
                                    rotation_vote="word", char_boxes=False, polys=None, points=None, max_windows=1,
                                    windows=None, language_model=None, pattern=None, char_scores=False,
                                    char_alternatives=0, hotwords=None):
        """images_t (N,H,W,3) u8 CUDA; boxes (N,M,4,2) f32 CUDA; counts host ndarray -> labels (B,48) i32 CUDA
        (``with_scores``: (labels, logp (B,) f32 CUDA); ``beam_width`` / ``top_paths`` / ``lexicon`` /
        ``language_model`` / ``pattern`` / ``hotwords``: see ``predict_device``).

        ``rotations`` / ``rotation_vote`` (``check_rotations``): every box is cut and decoded once per listed turn, one
        turn after another (the CRNN workspace stays that of B crops), and ``b2o_select_rotation`` keeps one reading per
        word.  The result then ends with the chosen turns (B,) int32 CUDA: (labels, turns) or (labels, logp, turns), in
        the shapes of the call without rotations.  ``boxes`` and ``flat`` are rolled in place to start at the chosen
        turn's corner: box[0] is the text's own top-left corner.

        ``char_boxes=True``: the result also ends with every reading's characters, spans (B,48,2) int32 -- each
        character's first and last emitting step (``b2o_ctc_align``), -1 past the last -- and cells (B,48,4,2) float32,
        its quad in detector-input pixels (``b2o_char_cells``), NaN past the last character; (B,P,48,2) / (B,P,48,4,2)
        with ``top_paths = P > 1``.

        ``char_scores=True`` (``check_char_scores``, with ``char_alternatives``): the result ends with every reading's
        character confidences (B,48) float32 (``b2o_crnn_char_scores``) and, with ``char_alternatives = A > 0``, its
        alternatives' labels (B,48,A) int32 and posteriors (B,48,A) float32, after the spans and cells when both are
        asked for; (B,P,48) / (B,P,48,A) with ``top_paths = P > 1``.  It combines with every decoder, rotations and
        polygons.

        Optional device-side by-products of the earlier stages, so that nothing but the kernel launches is
        left to do once the host knows the counts: ``gray`` (N,H,W) u8 from ``b2o_resize_pad_batch``;
        ``flat`` (>=B,4,2) / ``image_index`` (>=B,) from ``b2o_compact_boxes``.

        ``polys`` (>=B,18,2) float32 / ``points`` (>=B,) int32 CUDA, the dense polygons of ``b2o_compact_polys`` in the
        order of ``flat`` (with ``image_index``): every word is read along its polygon (``b2o_warp_polys``); a 4-point
        entry reads as its box.  Rotations and character cells do not combine with polygons (``ValueError``).

        ``max_windows`` (``check_windows``): every box wider than the crop at full height is read in up to that many
        windows (``b2o_warp_windows``, ``b2o_stitch_windows``); labels are then (B,48 max_windows), -1 padded, or
        (B,48) as without the option when no box is wide.  ``windows``: host ints (B,), the K of every box as
        ``b2o_window_counts`` gives them (``Pipeline.recognize`` reads them back with the box counts; ``ValueError`` for
        another shape or a count outside [1, max_windows]); None: computed here and read back, one more
        synchronisation."""
        lexicon, pattern, hotwords = self._decoder(beam_width, top_paths, lexicon, language_model, pattern, hotwords)
        turns = check_rotations(rotations, rotation_vote)
        scores = check_char_scores(char_scores, char_alternatives)
        max_windows = check_windows(max_windows, beam_width, lexicon, turns, char_boxes, polys is not None,
                                    scores is not None)
        if polys is not None and (turns is not None or char_boxes):
            raise ValueError("polygons do not combine with rotations or character boxes")
        counts = np.asarray(counts)
        m = boxes.shape[1]
        total = int(np.minimum(counts, m).sum())
        if max_windows > 1 and windows is not None:
            windows = np.asarray(windows)
            if (windows.shape != (total,) or not np.issubdtype(windows.dtype, np.integer)
                    or (total and (windows.min() < 1 or windows.max() > max_windows))):
                raise ValueError(f"windows must hold one window count in [1, {max_windows}] per box ({total}), as "
                                 f"b2o_window_counts gives them; got shape {windows.shape}")
        if total == 0:
            parts = (1 + bool(with_scores) + (turns is not None) + 2 * bool(char_boxes)
                     + (0 if scores is None else 1 + 2 * bool(scores)))
            return None if parts == 1 else (None,) * parts
        if self.color:
            gray = images_t                                       # color recognizer: crops come straight from the RGB batch
        elif gray is None:
            gray = self.gray_device(images_t)
        if flat is None or image_index is None:
            n = len(counts)
            flat = torch.empty((n * m, 4, 2), dtype=torch.float32, device=self.device)
            image_index = torch.empty((n * m,), dtype=torch.int32, device=self.device)
            counts_dev = torch.from_numpy(counts.astype(np.int32)).to(self.device)
            self.ctx.compact_boxes(boxes.data_ptr(), counts_dev.data_ptr(), n, m, flat.data_ptr(),
                                   image_index.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
        if max_windows > 1:
            labels, logp = self._read_windowed(gray, flat[:total], image_index[:total], max_windows, windows,
                                               with_scores)
            return (labels, logp) if with_scores else labels
        if polys is not None:
            crnn_in, _ = self.warp_polys_device(gray, polys[:total], points[:total], image_index[:total])
            return self.predict_device(crnn_in, with_scores=with_scores, beam_width=beam_width, top_paths=top_paths,
                                       lexicon=lexicon, language_model=language_model, pattern=pattern,
                                       char_scores=scores, hotwords=hotwords)
        if turns is not None:
            return self._recognize_turns(gray, flat[:total], image_index[:total], len(counts), boxes, turns,
                                         rotation_vote, with_scores, beam_width, top_paths, lexicon, char_boxes,
                                         language_model, pattern, scores, hotwords)
        if char_boxes:
            labels, logp, spans, cells, *extra = self._read_cells(gray, flat[:total], image_index[:total], beam_width,
                                                                  top_paths, lexicon, language_model, pattern, scores,
                                                                  hotwords)
            return ((labels, logp, spans, cells) if with_scores else (labels, spans, cells)) + tuple(extra)
        crnn_in, _ = self.warp_device(gray, flat[:total], image_index[:total])
        return self.predict_device(crnn_in, with_scores=with_scores, beam_width=beam_width, top_paths=top_paths,
                                   lexicon=lexicon, language_model=language_model, pattern=pattern, char_scores=scores,
                                   hotwords=hotwords)

    def _read_cells(self, gray, flat, image_index, beam_width, top_paths, lexicon, language_model=None, pattern=None,
                    char_scores=None, hotwords=None):
        """Warp + CRNN + decoder + alignment + cells of one pass: (labels, logp, spans, cells) in the shapes of
        ``recognize_from_boxes_device``, followed by the character scores with ``char_scores`` = A."""
        crnn_in, _ = self.warp_device(gray, flat, image_index)
        labels, logp, spans, theta, *scores = self._predict_aligned(crnn_in, beam_width, top_paths, lexicon,
                                                                    language_model, pattern, char_scores, hotwords)
        cells = self.char_cells_device(spans, theta, flat)
        out = (labels, logp, spans, cells) + (tuple(t for t in scores[0] if t is not None) if scores else ())
        return tuple(t[:, 0] for t in out) if top_paths == 1 else out

    def _recognize_turns(self, gray, flat, image_index, n_images, table, turns, vote, with_scores, beam_width,
                         top_paths, lexicon, char_boxes=False, language_model=None, pattern=None, char_scores=None,
                         hotwords=None):
        """Warp + CRNN + decoder for each turn into its slot of one (R,B,P,48) / (R,B,P) stack, then
        ``b2o_select_rotation``, which also rolls ``flat`` and ``table`` (None: no table) in place.  ``char_boxes``: each
        turn's spans and theta are stacked alike, and the chosen turn's cells are built from the boxes as they were cut.
        With ``language_model`` or ``hotwords`` the vote compares the readings' F_end, and the chosen turn's acoustic
        logp is gathered on the device.  ``char_scores`` = A: each turn's character scores are stacked alike and the chosen turn's
        gathered; they end the result."""
        b, p, r = flat.shape[0], int(top_paths), len(turns)
        labels_all = torch.empty((r, b, p, STEPS), dtype=torch.int32, device=self.device)
        logp_all = torch.empty((r, b, p), dtype=torch.float32, device=self.device)
        fused = language_model is not None or hotwords is not None
        fused_all = torch.empty((r, b, p), dtype=torch.float32, device=self.device) if fused else None
        spans_all = theta_all = cut = None
        if char_boxes:
            spans_all = torch.empty((r, b, p, STEPS, 2), dtype=torch.int32, device=self.device)
            theta_all = torch.empty((r, b, 6), dtype=torch.float32, device=self.device) if self.stn else None
            cut = flat.clone()                           # b2o_select_rotation rolls flat in place
        scores_all = None if char_scores is None else self._score_buffers((r, b, p), char_scores)
        for j, turn in enumerate(turns):
            crnn_in, _ = self.warp_device(gray, flat, image_index, turn=turn)
            self._forward(crnn_in, labels_all[j], logp_all[j], beam_width, p, lexicon,
                          None if spans_all is None else spans_all[j], None if theta_all is None else theta_all[j],
                          language_model, None if fused_all is None else fused_all[j], pattern,
                          None if scores_all is None else tuple(None if t is None else t[j] for t in scores_all),
                          hotwords)
        labels = torch.empty((b, p, STEPS), dtype=torch.int32, device=self.device)
        logp = torch.empty((b, p), dtype=torch.float32, device=self.device)
        chosen = torch.empty((b,), dtype=torch.int32, device=self.device)
        vote_logp = logp_all if fused_all is None else fused_all
        self.ctx.select_rotation(labels_all.data_ptr(), vote_logp.data_ptr(), image_index.data_ptr(), n_images, b, p,
                                 turns, ROTATION_VOTES[vote], labels.data_ptr(), logp.data_ptr(), chosen.data_ptr(),
                                 flat.data_ptr(), None if table is None else table.data_ptr(),
                                 0 if table is None else table.shape[1], torch.cuda.current_stream(self.device).cuda_stream)
        extra = ()
        if char_boxes or fused_all is not None or scores_all is not None:
            slot = torch.zeros(4, dtype=torch.int64, device=self.device)
            slot[list(turns)] = torch.arange(r, device=self.device)
            pick, rows = slot[chosen.long()], torch.arange(b, device=self.device)
        if fused_all is not None:
            logp = logp_all[pick, rows]                  # the vote ran on F_end; the readings keep their acoustic logp
        if char_boxes:
            spans = spans_all[pick, rows]
            cells = self.char_cells_device(spans, None if theta_all is None else theta_all[pick, rows], cut, chosen)
            extra = (spans[:, 0], cells[:, 0]) if p == 1 else (spans, cells)
        if scores_all is not None:
            picked = tuple(t[pick, rows] for t in scores_all if t is not None)
            extra = extra + (tuple(t[:, 0] for t in picked) if p == 1 else picked)
        if p == 1:
            labels, logp = labels.view(b, STEPS), logp.view(b)
        return ((labels, logp, chosen) if with_scores else (labels, chosen)) + extra

    # ------------------------------------------------------------------ reference API
    def recognize_from_boxes(self, images, box_groups, return_scores=False, beam_width=None, top_paths=1, lexicon=None,
                             rotations=None, rotation_vote="word", return_char_boxes=False, max_windows=1,
                             language_model=None, pattern=None, return_char_scores=False, char_alternatives=0,
                             hotwords=None, **kwargs) -> typing.List[typing.List[str]]:
        """Same contract as reference recognition.py:491-537.  ``return_scores=True``: every word is a
        (text, confidence) pair instead, see ``confidences``.  ``beam_width`` / ``top_paths`` / ``lexicon`` /
        ``language_model`` / ``pattern`` / ``hotwords``: as ``recognize_crops``; with rotations the vote compares the fused scores F_end of a language model or hotwords.  ``rotations`` / ``rotation_vote``: every box is read in each listed quarter turn and the
        most probable reading kept, per word or per image (one box group), see ``check_rotations``.
        ``return_char_boxes=True``: every word is a tuple that ends with its character cells, an (n,4,2) float32 array
        of quads in the image's pixels for a text of n characters (a list of P arrays with ``top_paths = P > 1``):
        (text, cells) or (text, confidence, cells); see ``recognize_from_boxes_device``.
        ``return_char_scores=True`` / ``char_alternatives``: every word's tuple ends with its character scores, after
        the cells when both are asked for, as ``recognize_crops`` returns them.

        A box group may also hold polygons, (2m,2) arrays with 3 <= m <= 9 as ``Detector.detect(return_polygons=True)``
        returns them (``check_polygons``): such a word is read along its polygon (``b2o_warp_polys``), a 4-point entry
        of the same group exactly as without polygons.  Rotations and character boxes do not combine with polygons
        (``ValueError``).
        ``max_windows``: every box wider than the 200 x 31 crop at full height is read in up to that many overlapping
        windows and their steps stitched into one reading (``check_windows``; greedy decoding, boxes only)."""
        lexicon, pattern, hotwords = self._decoder(beam_width, top_paths, lexicon, language_model, pattern, hotwords)
        turns = check_rotations(rotations, rotation_vote)
        assert len(box_groups) == len(images), "You must provide the same number of box groups as images."
        from .detection import _as_device_images

        entries = [e for g in box_groups for e in g]
        polygons = any(np.ndim(e) == 2 and np.shape(e)[0] != 4 for e in entries)
        char_scores = check_char_scores(return_char_scores, char_alternatives)
        max_windows = check_windows(max_windows, beam_width, lexicon, turns, return_char_boxes, polygons,
                                    char_scores is not None)
        if polygons:
            return self._recognize_polygons(images, box_groups, entries, return_scores, turns, return_char_boxes,
                                            beam_width, top_paths, lexicon, language_model, pattern, char_scores,
                                            hotwords)
        images_t = _as_device_images(images, self.device)
        counts = np.array([len(b) for b in box_groups], dtype=np.int64)
        if counts.sum() == 0:
            return [[]] * len(images)
        flat = np.concatenate([np.asarray(b, dtype=np.float32).reshape(-1, 4, 2) for b in box_groups if len(b)])
        # caller-supplied quads: tools.warpBox first replaces each by its minimum rotated rectangle and divides by its
        # truncated width / height (tools.py:88-95; ZeroDivisionError for a degenerate box).  Rectangles -- everything
        # a Detector returns -- pass through bit for bit.
        flat = tools.rectify_boxes(flat)
        flat_t = torch.from_numpy(np.ascontiguousarray(flat)).to(self.device)
        idx = torch.from_numpy(np.repeat(np.arange(len(counts), dtype=np.int32), counts)).to(self.device)
        gray = images_t if self.color else self.gray_device(images_t)
        beam = {"beam_width": beam_width, "top_paths": top_paths, "lexicon": lexicon, "language_model": language_model,
                "pattern": pattern, "hotwords": hotwords}
        if return_char_boxes or char_scores is not None:
            cells = None
            if turns is not None:
                labels, logp, _, *rest = self._recognize_turns(gray, flat_t, idx, len(counts), None, turns,
                                                               rotation_vote, True, char_boxes=return_char_boxes,
                                                               char_scores=char_scores, **beam)
                if return_char_boxes:
                    cells, rest = rest[1], rest[2:]
            elif return_char_boxes:
                labels, logp, _, cells, *rest = self._read_cells(gray, flat_t, idx, char_scores=char_scores, **beam)
            else:
                crnn_in, _ = self.warp_device(gray, flat_t, idx)
                labels, logp, *rest = self.predict_device(crnn_in, with_scores=True, char_scores=char_scores, **beam)
            predictions = self._host_words(labels, logp, top_paths, return_scores, cells,
                                           rest if char_scores is not None else None)
        elif turns is not None:
            labels, logp, _ = self._recognize_turns(gray, flat_t, idx, len(counts), None, turns, rotation_vote, True,
                                                    **beam)
            texts, conf = decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())
            predictions = list(zip(texts, conf)) if return_scores else texts
        elif max_windows > 1:
            labels, logp = self._read_windowed(gray, flat_t, idx, max_windows, None, True)
            texts, conf = decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())
            predictions = list(zip(texts, conf)) if return_scores else texts
        elif return_scores:
            crnn_in, _ = self.warp_device(gray, flat_t, idx)
            labels, logp = self.predict_device(crnn_in, with_scores=True, **beam)
            predictions = list(zip(*decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())))
        else:
            crnn_in, _ = self.warp_device(gray, flat_t, idx)
            predictions = decode_paths(self.predict_device(crnn_in, **beam).cpu().numpy(), self.alphabet)[0]
        ends = np.cumsum(counts)
        return [predictions[int(e - c):int(e)] for c, e in zip(counts, ends)]

    def _recognize_polygons(self, images, box_groups, entries, return_scores, turns, char_boxes, beam_width, top_paths,
                            lexicon, language_model=None, pattern=None, char_scores=None, hotwords=None):
        """``recognize_from_boxes`` for box groups that hold polygons: 4-point entries are rectified as
        ``tools.rectify_boxes`` does and cut as boxes, the others along their polygon, all in one ``b2o_warp_polys``."""
        if turns is not None or char_boxes:
            raise ValueError("polygons do not combine with rotations or return_char_boxes")
        polys, points = check_polygons(entries)
        four = points == 4
        if four.any():
            polys[four, :4] = tools.rectify_boxes(polys[four, :4])
        from .detection import _as_device_images

        images_t = _as_device_images(images, self.device)
        counts = np.array([len(b) for b in box_groups], dtype=np.int64)
        idx = torch.from_numpy(np.repeat(np.arange(len(counts), dtype=np.int32), counts)).to(self.device)
        gray = images_t if self.color else self.gray_device(images_t)
        crnn_in, _ = self.warp_polys_device(gray, torch.from_numpy(polys).to(self.device),
                                            torch.from_numpy(points).to(self.device), idx)
        beam = {"beam_width": beam_width, "top_paths": top_paths, "lexicon": lexicon, "language_model": language_model,
                "pattern": pattern, "hotwords": hotwords}
        if char_scores is not None:
            labels, logp, *scores = self.predict_device(crnn_in, with_scores=True, char_scores=char_scores, **beam)
            predictions = self._host_words(labels, logp, top_paths, return_scores, None, scores)
        elif return_scores:
            labels, logp = self.predict_device(crnn_in, with_scores=True, **beam)
            predictions = list(zip(*decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())))
        else:
            predictions = decode_paths(self.predict_device(crnn_in, **beam).cpu().numpy(), self.alphabet)[0]
        ends = np.cumsum(counts)
        return [predictions[int(e - c):int(e)] for c, e in zip(counts, ends)]

    # ------------------------------------------------------------------ training the top layer
    def _input_crops(self, crops, what):
        """(N,31,200[,3]) uint8 crops -> the CRNN input (N,200,31[,3]) fp16 on the device."""
        tail = (3,) if self.color else ()
        shape = tuple(crops.shape) if hasattr(crops, "shape") else None
        dtype_ok = (crops.dtype == torch.uint8) if isinstance(crops, torch.Tensor) else (np.asarray(crops).dtype == np.uint8)
        if shape is None or shape[1:] != (TARGET_HEIGHT, TARGET_WIDTH) + tail or not dtype_ok:
            raise ValueError(f"{what} must be a uint8 array of shape (N, {TARGET_HEIGHT}, {TARGET_WIDTH}"
                             f"{', 3' if self.color else ''}), got {shape}")
        return crops

    def _features(self, crops, chunk=512, sequence=False):
        """``b2o_crnn_features`` of every crop, in chunks that bound the CRNN workspace: (N,48,256) fp16 CUDA; with
        ``sequence``, ``b2o_crnn_sequence_features`` (fc_9's output): (N,50,128)."""
        n = int(crops.shape[0])
        feats = torch.empty((n,) + ((50, 128) if sequence else (STEPS, 256)), dtype=torch.float16, device=self.device)
        run = self.ctx.crnn_sequence_features if sequence else self.ctx.crnn_features
        stream = torch.cuda.current_stream(self.device).cuda_stream
        nbytes = self.ctx.crnn_workspace_bytes(min(chunk, n))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        tail = (3,) if self.color else ()
        for i in range(0, n, chunk):
            part = crops[i:i + chunk]
            t = part if isinstance(part, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(part))
            t = t.to(self.device).contiguous()
            b = t.shape[0]
            x = torch.empty((b, TARGET_WIDTH, TARGET_HEIGHT) + tail, dtype=torch.float16, device=self.device)
            self.ctx.crops_to_input(t.data_ptr(), b, x.data_ptr(), stream, color=self.color)
            run(x.data_ptr(), b, feats[i:i + b].data_ptr(), ws.data_ptr(), nbytes, stream)
        return feats

    def _batch_targets(self, offsets, labels, idx):
        """The CSR targets of rows ``idx`` of a CSR set, on the device."""
        lengths = np.diff(offsets)[idx]
        off = np.zeros(len(idx) + 1, np.int32)
        off[1:] = np.cumsum(lengths)
        lab = np.concatenate([labels[offsets[j]:offsets[j + 1]] for j in idx]).astype(np.int16)
        return torch.from_numpy(off).to(self.device), torch.from_numpy(lab).to(self.device)

    def _mean_loss(self, feats, offsets, labels, w, bias, chunk=1024):
        """Mean of L_b over a feature set, without dropout (``b2o_ctc_loss_grad``, loss only), in fp64 on the host."""
        n, k = feats.shape[0], w.shape[1]
        loss = torch.empty(n, dtype=torch.float32, device=self.device)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        for i in range(0, n, chunk):
            idx = np.arange(i, min(n, i + chunk), dtype=np.int32)
            off, lab = self._batch_targets(offsets, labels, idx)
            index = torch.from_numpy(idx).to(self.device)
            self.ctx.ctc_loss_grad(feats.data_ptr(), n, index.data_ptr(), len(idx), k, w.data_ptr(), bias.data_ptr(),
                                   off.data_ptr(), lab.data_ptr(), 0.0, 0, 0, loss[i:].data_ptr(), None, None, None,
                                   None, 0, stream)
        return float(loss.cpu().numpy().astype(np.float64).mean())

    def _fit_args(self, crops, texts, epochs, batch_size, learning_rate, dropout, seed, validation):
        """The argument checks of ``fit_top`` and ``fit_recurrent``, all made before anything runs on the device:
        (CSR offsets, labels, N, crops, validation as (crops, offsets, labels) or None)."""
        def is_int(v):
            return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))
        offsets, labels = check_texts(texts, self.alphabet)
        n = len(offsets) - 1
        crops = self._input_crops(crops, "crops")
        if crops.shape[0] != n:
            raise ValueError(f"{crops.shape[0]} crops but {n} texts")
        if not is_int(epochs) or epochs < 1:
            raise ValueError(f"epochs must be an int >= 1, got {epochs!r}")
        if not is_int(batch_size) or batch_size < 1:
            raise ValueError(f"batch_size must be an int >= 1, got {batch_size!r}")
        if not is_int(seed) or seed < 0:
            raise ValueError(f"seed must be an int >= 0, got {seed!r}")
        if not (isinstance(learning_rate, (int, float)) and learning_rate > 0):
            raise ValueError(f"learning_rate must be a positive number, got {learning_rate!r}")
        if not (isinstance(dropout, (int, float)) and 0 <= dropout < 1):
            raise ValueError(f"dropout must be in [0, 1), got {dropout!r}")
        val = None
        if validation is not None:
            if not isinstance(validation, (tuple, list)) or len(validation) != 2:
                raise ValueError("validation must be a (crops, texts) pair")
            v_off, v_lab = check_texts(validation[1], self.alphabet)
            v_crops = self._input_crops(validation[0], "validation crops")
            if v_crops.shape[0] != len(v_off) - 1:
                raise ValueError(f"{v_crops.shape[0]} validation crops but {len(v_off) - 1} texts")
            val = (v_crops, v_off, v_lab)
        return offsets, labels, n, crops, val

    def fit_top(self, crops, texts, epochs=1, batch_size=64, learning_rate=1e-3, dropout=0.25, seed=0, validation=None):
        """Train the output layer (``fc_12``, Dense 256 -> len(alphabet) + 1 with bias) on labelled word crops, the rest
        of the CRNN frozen -- the reference's fine-tuning workflow (``compile()`` + ``training_model``,
        recognition.py:334-349, 539-545) restricted to the top.  ``crops``: (N,31,200) uint8 -- (N,31,200,3) for a color
        recognizer -- as ``recognize_crops`` takes them; ``texts``: N strings over the alphabet (``check_texts``).
        ``validation``: an optional (crops, texts) pair.

        The BiLSTM features of every crop are computed once (``b2o_crnn_features``) and kept on the device, 24.6 kB per
        crop.  Each epoch shuffles them with ``np.random.default_rng(seed)`` and runs, per batch, the Keras
        ``ctc_batch_cost`` loss and its gradient (``b2o_ctc_loss_grad``; Dropout(``dropout``) before the layer, as in
        the reference's graph) and one RMSprop step (``b2o_rmsprop_step``, Keras' defaults rho 0.9, eps 1e-7).  Training
        starts from the current top: the re-initialised one for a new alphabet, the checkpoint's otherwise.  At the end
        the new top is installed (``b2o_crnn_set_top``), so every recognition path uses it.  Same seed and inputs give
        bit-identical weights.

        Returns {"loss": [...], "val_loss": [...]}: per epoch the mean L_b over the training crops (as they were seen,
        with dropout) and over the validation crops (without dropout, after the epoch; empty without ``validation``)."""
        offsets, labels, n, crops, val = self._fit_args(crops, texts, epochs, batch_size, learning_rate, dropout, seed,
                                                        validation)
        k = len(self.alphabet) + 1
        stream = torch.cuda.current_stream(self.device).cuda_stream
        feats = self._features(crops)
        v_feats = self._features(val[0]) if val is not None else None
        w = torch.from_numpy(np.ascontiguousarray(self._tensors["fc_12.kernel"], np.float32)).to(self.device)
        bias = torch.from_numpy(np.ascontiguousarray(self._tensors["fc_12.bias"], np.float32)).to(self.device)
        acc_w, acc_b = torch.zeros_like(w), torch.zeros_like(bias)
        grad_w, grad_b = torch.empty_like(w), torch.empty_like(bias)
        bs = min(int(batch_size), n)
        nbytes = self.ctx.ctc_train_workspace_bytes(bs, k)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        loss = torch.empty(n, dtype=torch.float32, device=self.device)
        rng = np.random.default_rng(seed)
        history = {"loss": [], "val_loss": []}
        step = 0
        for _ in range(epochs):
            perm = rng.permutation(n).astype(np.int32)
            for i in range(0, n, bs):
                idx = perm[i:i + bs]
                off, lab = self._batch_targets(offsets, labels, idx)
                index = torch.from_numpy(idx).to(self.device)
                self.ctx.ctc_loss_grad(feats.data_ptr(), n, index.data_ptr(), len(idx), k, w.data_ptr(),
                                       bias.data_ptr(), off.data_ptr(), lab.data_ptr(), dropout, seed, step,
                                       loss[i:].data_ptr(), grad_w.data_ptr(), grad_b.data_ptr(), None, ws.data_ptr(),
                                       nbytes, stream)
                self.ctx.rmsprop_step(w.data_ptr(), grad_w.data_ptr(), acc_w.data_ptr(), w.numel(), learning_rate, 0.9,
                                      1e-7, stream)
                self.ctx.rmsprop_step(bias.data_ptr(), grad_b.data_ptr(), acc_b.data_ptr(), bias.numel(),
                                      learning_rate, 0.9, 1e-7, stream)
                step += 1
            history["loss"].append(float(loss.cpu().numpy().astype(np.float64).mean()))
            if val is not None:
                history["val_loss"].append(self._mean_loss(v_feats, val[1], val[2], w, bias))
        self.ctx.crnn_set_top(w.data_ptr(), bias.data_ptr(), k, stream)
        self._tensors = dict(self._tensors)
        self._tensors["fc_12.kernel"] = w.cpu().numpy()
        self._tensors["fc_12.bias"] = bias.cpu().numpy()
        return history

    # ------------------------------------------------------------------ fine-tuning the recurrent head
    RNN_LAYERS = ("lstm_10", "lstm_10_back", "lstm_11", "lstm_11_back")
    _RNN_PARTS = (("kernel", (128, 512)), ("recurrent_kernel", (128, 512)), ("bias", (512,)))

    def _rnn_tensor_names(self):
        """The 14 tensors ``fit_recurrent`` trains, in the order of ``b2o_rnn_loss_grad``'s parameter vector."""
        k = len(self.alphabet) + 1
        names = [(f"{layer}.{part}", shape) for layer in self.RNN_LAYERS for part, shape in self._RNN_PARTS]
        return names + [("fc_12.kernel", (256, k)), ("fc_12.bias", (k,))]

    def fit_recurrent(self, crops, texts, epochs=1, batch_size=64, learning_rate=1e-3, dropout=0.25, seed=0,
                      validation=None):
        """Fine-tune the BiLSTM (``lstm_10``, ``lstm_10_back``, ``lstm_11``, ``lstm_11_back``: kernel, recurrent kernel
        and bias of each) together with the output layer ``fc_12`` -- the reference's fine-tuning workflow
        (``compile()`` + ``training_model``, recognition.py:334-349, 539-545) with the convolutions, the STN and
        ``fc_9`` frozen.  Arguments, checks and the returned history are those of ``fit_top``.

        The ``fc_9`` output of every crop is computed once (``b2o_crnn_sequence_features``) and kept on the device,
        12.8 kB per crop.  Each batch runs the BiLSTM forward with the inference arithmetic, the CTC loss and
        backpropagation through time (``b2o_rnn_loss_grad``), then one Keras RMSprop step (momentum 0, rho 0.9,
        eps 1e-7) on fp32 master weights of all 14 tensors (``b2o_rmsprop_step``).  At the end the trained tensors
        replace this recognizer's and the CRNN is reloaded from them, so it equals ``Recognizer(alphabet,
        weights=<save_weights file>)`` bit for bit.  Same seed and inputs give bit-identical weights."""
        offsets, labels, n, crops, val = self._fit_args(crops, texts, epochs, batch_size, learning_rate, dropout, seed,
                                                        validation)
        k = len(self.alphabet) + 1
        stream = torch.cuda.current_stream(self.device).cuda_stream
        seq = self._features(crops, sequence=True)
        v_seq = self._features(val[0], sequence=True) if val is not None else None
        names = self._rnn_tensor_names()
        params = torch.from_numpy(np.concatenate(
            [np.ascontiguousarray(self._tensors[name], np.float32).reshape(-1) for name, _ in names])).to(self.device)
        acc, grad = torch.zeros_like(params), torch.empty_like(params)
        bs = min(int(batch_size), n)
        nbytes = self.ctx.rnn_train_workspace_bytes(bs, k)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        loss = torch.empty(n, dtype=torch.float32, device=self.device)

        def mean_loss(x, off, lab):
            m = x.shape[0]
            out = torch.empty(m, dtype=torch.float32, device=self.device)
            for i in range(0, m, bs):
                idx = np.arange(i, min(m, i + bs), dtype=np.int32)
                o, lb = self._batch_targets(off, lab, idx)
                index = torch.from_numpy(idx).to(self.device)
                self.ctx.rnn_loss_grad(x.data_ptr(), m, index.data_ptr(), len(idx), k, params.data_ptr(), o.data_ptr(),
                                       lb.data_ptr(), 0.0, 0, 0, out[i:].data_ptr(), None, ws.data_ptr(), nbytes, stream)
            return float(out.cpu().numpy().astype(np.float64).mean())

        rng = np.random.default_rng(seed)
        history = {"loss": [], "val_loss": []}
        step = 0
        for _ in range(epochs):
            perm = rng.permutation(n).astype(np.int32)
            for i in range(0, n, bs):
                idx = perm[i:i + bs]
                off, lab = self._batch_targets(offsets, labels, idx)
                index = torch.from_numpy(idx).to(self.device)
                self.ctx.rnn_loss_grad(seq.data_ptr(), n, index.data_ptr(), len(idx), k, params.data_ptr(),
                                       off.data_ptr(), lab.data_ptr(), dropout, seed, step, loss[i:].data_ptr(),
                                       grad.data_ptr(), ws.data_ptr(), nbytes, stream)
                self.ctx.rmsprop_step(params.data_ptr(), grad.data_ptr(), acc.data_ptr(), params.numel(), learning_rate,
                                      0.9, 1e-7, stream)
                step += 1
            history["loss"].append(float(loss.cpu().numpy().astype(np.float64).mean()))
            if val is not None:
                history["val_loss"].append(mean_loss(v_seq, val[1], val[2]))
        host = params.cpu().numpy()
        tensors, at = dict(self._tensors), 0
        for name, shape in names:
            size = int(np.prod(shape))
            tensors[name] = host[at:at + size].reshape(shape).copy()
            at += size
        self.ctx.load_crnn(tensors)
        self._tensors = tensors
        return history

    def save_weights(self, path):
        """Every CRNN tensor of this recognizer -- with the top ``fit_top`` trained -- as a flat ``.npz`` keyed like
        ``weights.py``, which ``Recognizer(alphabet, weights=path)`` loads unchanged."""
        np.savez(path, **{name: np.asarray(v, dtype=np.float32) for name, v in self._tensors.items()})
