"""The derivation behind csrc/hf_pretok.cuh, as an executable check: for both pre-tokenizer patterns the
position-local rules the warp evaluates in parallel (one char back, one ahead, plus the three scanned facts of
pattern 2) give exactly the token starts of the leftmost-first sequential regex scan that the oracle restates
(oracle/hf_bpe_oracle.cc gpt2_split / cl100k_split, themselves pinned to pip `tokenizers`).  Pure Python, seconds."""
import random

O, L, N, S = 0, 1, 2, 3
WS = " \t\n\r\x0b\x0c\x85\xa0　 "


def cls(ch):
    if ch in WS:
        return S
    if ch.isalpha():
        return L
    if ch.isdigit():
        return N
    return O


def fold(ch):
    return ch.lower() if "A" <= ch <= "Z" else ("s" if ch == "ſ" else ch)


def contraction(c, i, ci):
    n = len(c)
    f = (lambda k: fold(c[k]) if k < n else "") if ci else (lambda k: c[k] if k < n else "")
    if c[i] != "'":
        return 0
    if f(i + 1) != "" and f(i + 1) in "stmd":
        return 2
    if f(i + 1) + f(i + 2) in ("re", "ve", "ll"):
        return 3
    return 0


# ---------------------------------------------------------------- pattern 1 (GPT-2)
def seq1(c):
    n, k, i, out = len(c), [cls(x) for x in c], 0, []
    while i < n:
        j = i + contraction(c, i, False)
        if j == i:
            s = i + 1 if (c[i] == " " and i + 1 < n and k[i + 1] != S) else i
            if k[s] != S:
                j = s
                while j < n and k[j] == k[s]:
                    j += 1
        if j == i:
            e = i
            while e < n and k[e] == S:
                e += 1
            j = e if e == n else (e - 1 if e - i >= 2 else e)
        out.append(i)
        i = j
    return out


def rules1(c):
    n, k = len(c), [cls(x) for x in c]
    clen = [contraction(c, p, False) if c[p] == "'" and (p == 0 or (k[p - 1] != O and c[p - 1] != " ")) else 0
            for p in range(n)]
    out = []
    for p in range(n):
        if p == 0 or clen[p]:
            st = True
        else:
            c1, c2, c3 = clen[p - 1], clen[p - 2] if p >= 2 else 0, clen[p - 3] if p >= 3 else 0
            if c1 or c2 == 3:
                st = False
            elif c2 == 2 or c3 == 3:
                st = True
            else:
                a, b = k[p - 1], k[p]
                if b == S:
                    st = a != S or (p + 1 < n and k[p + 1] != S)
                else:
                    st = (c[p - 1] != " ") if a == S else a != b
        if st:
            out.append(p)
    return out


# ---------------------------------------------------------------- pattern 2 (cl100k family, K digits)
def seq2(c, K):
    n, k, i, out = len(c), [cls(x) for x in c], 0, []
    nl = lambda x: x in "\r\n"  # noqa: E731
    while i < n:
        j = i + contraction(c, i, True)
        if j == i:
            s = i + 1 if (k[i] not in (L, N) and not nl(c[i]) and i + 1 < n and k[i + 1] == L) else i
            if k[s] == L:
                j = s
                while j < n and k[j] == L:
                    j += 1
        if j == i and k[i] == N:
            while j < n and k[j] == N and j - i < K:
                j += 1
        if j == i:
            s = i + 1 if (c[i] == " " and i + 1 < n and k[i + 1] == O) else i
            if k[s] == O:
                j = s
                while j < n and k[j] == O:
                    j += 1
                while j < n and nl(c[j]):
                    j += 1
        if j == i:
            e = i
            while e < n and k[e] == S:
                e += 1
            last = max([t for t in range(i, e) if nl(c[t])], default=-1)
            j = last + 1 if last >= 0 else (e if e == n else (e - 1 if e - i >= 2 else e))
        out.append(i)
        i = j
    return out


def rules2(c, K):
    n, k = len(c), [cls(x) for x in c]
    nl = [x in "\r\n" for x in c]
    s_o = lambda i: i == 0 or (k[i - 1] != O and c[i - 1] != " ")  # noqa: E731  a punctuation char that starts a token
    clen = [contraction(c, i, True) if c[i] == "'" and s_o(i) else 0 for i in range(n)]
    sw, ds, hna, cnt = [False] * n, [False] * n, [False] * n, 0
    for i in range(n):
        if nl[i]:                                   # C1: CR/LF swallowed by a punctuation run's [\r\n]* tail
            j = i - 1
            while j >= 0 and nl[j]:
                j -= 1
            sw[i] = j >= 0 and k[j] == O
        if k[i] == N:                               # C1: digit index inside its run
            ds[i] = cnt % K == 0
            cnt += 1
        else:
            cnt = 0
        if k[i] == S and not nl[i]:                 # C2: a CR/LF still ahead in the whitespace run
            j = i + 1
            while j < n and k[j] == S:
                if nl[j]:
                    hna[i] = True
                    break
                j += 1
    out = []
    for i in range(n):
        if i == 0 or clen[i]:
            st = True
        else:
            c1, c2, c3 = clen[i - 1], clen[i - 2] if i >= 2 else 0, clen[i - 3] if i >= 3 else 0
            if c1 or c2 == 3:
                st = False
            elif c2 == 2 or c3 == 3:
                st = True
            else:
                a, b = k[i - 1], k[i]
                if b == L:
                    st = False if a == L else (True if a == N else (nl[i - 1] if a == S else not s_o(i - 1)))
                elif b == N:
                    st = ds[i]
                elif b == O:
                    st = s_o(i)
                elif nl[i]:
                    st = (not sw[i]) and a != S
                elif hna[i]:
                    st = a != S or (nl[i - 1] and sw[i - 1])
                else:
                    st = a != S or nl[i - 1] or (i + 1 < n and k[i + 1] != S)
        if st:
            out.append(i)
    return out


ALPHA = list("ab  \t\n\r''.!12") + ["'s", "'RE", " '", "'ll", "é", " ", "　", "'ſ", "\n\n", "!\n", " \n", "'S"]


def test_gpt2_rules_equal_the_sequential_scan():
    rnd = random.Random(1)
    for _ in range(60000):
        s = "".join(rnd.choice(ALPHA) for _ in range(rnd.randrange(0, 14)))
        assert seq1(s) == rules1(s), repr(s)


def test_cl100k_rules_equal_the_sequential_scan():
    rnd = random.Random(5)
    for K in (1, 3):
        for _ in range(60000):
            s = "".join(rnd.choice(ALPHA) for _ in range(rnd.randrange(0, 14)))
            assert seq2(s, K) == rules2(s, K), (K, repr(s))


# ---------------------------------------------------------------- pattern 3 (DeepSeek-V3: three Isolated splits)
# kinds: LET = \p{L} or \p{M} outside the CJK ranges, NUM = \p{N}, CJK = [一-龥぀-ゟ゠-ヿ], WSP = whitespace,
#        PS = \p{P} or \p{S}, OTH = the rest (control / format / unassigned)
LET, NUM, CJK, WSP, PS, OTH = range(6)


def kind3(ch):
    import unicodedata
    cp = ord(ch)
    if 0x4E00 <= cp <= 0x9FA5 or 0x3040 <= cp <= 0x309F or 0x30A0 <= cp <= 0x30FF:
        return CJK
    if ch in WS:
        return WSP
    g = unicodedata.category(ch)[0]
    return {"L": LET, "M": LET, "N": NUM, "P": PS, "S": PS}.get(g, OTH)


def apunct(ch):
    return ch in "!\"#$%&'()*+,-./:;<=>?@[\\]^_`{|}~"


def aalpha(ch):
    return ("a" <= ch <= "z") or ("A" <= ch <= "Z")


def seq3(c):
    """sequential: split numbers (groups of 3), then CJK runs, then the main regex inside each remaining piece"""
    n, k, out = len(c), [kind3(x) for x in c], []
    nl = lambda x: x in "\r\n"  # noqa: E731

    def match_at(i, e):
        if apunct(c[i]) and i + 1 < e and aalpha(c[i + 1]):
            j = i + 2
            while j < e and aalpha(c[j]):
                j += 1
            return j
        s = i + 1 if (not nl(c[i]) and k[i] not in (LET, PS) and i + 1 < e and k[i + 1] == LET) else i
        if k[s] == LET:
            j = s
            while j < e and k[j] == LET:
                j += 1
            return j
        s = i + 1 if (c[i] == " " and i + 1 < e and k[i + 1] == PS) else i
        if k[s] == PS:
            j = s
            while j < e and k[j] == PS:
                j += 1
            while j < e and nl(c[j]):
                j += 1
            return j
        if k[i] == WSP:
            w = i
            while w < e and k[w] == WSP:
                w += 1
            last = max([t for t in range(i, w) if nl(c[t])], default=-1)
            return last + 1 if last >= 0 else (w if w == e else (w - 1 if w - i >= 2 else w))
        return i

    i = 0
    while i < n:
        if k[i] == NUM:
            j = i
            while j < n and k[j] == NUM and j - i < 3:
                j += 1
            out.append(i)
            i = j
            continue
        if k[i] == CJK:
            out.append(i)
            while i < n and k[i] == CJK:
                i += 1
            continue
        e = i
        while e < n and k[e] not in (NUM, CJK):
            e += 1
        t = i
        while t < e:
            j = match_at(t, e)
            out.append(t)
            if j > t:
                t = j
            else:
                t += 1
                while t < e and match_at(t, e) == t:
                    t += 1
        i = e
    return out


def rules3(c):
    """position-local rules + scanned facts (what csrc/hf_pretok.cuh hf_rules3 evaluates)"""
    n, k = len(c), [kind3(x) for x in c]
    nl = [x in "\r\n" for x in c]
    # an ASCII punctuation char that opens "punct + ASCII letters": it must be a token start itself (the previous char
    # is neither P/S — its run would have swallowed it — nor U+0020, which would be the " ?" prefix of a P/S run)
    ps_start = lambda i: i == 0 or (k[i - 1] != PS and c[i - 1] != " ")  # noqa: E731
    a_start = [apunct(c[i]) and i + 1 < n and aalpha(c[i + 1]) and ps_start(i) for i in range(n)]
    # scanned facts: CR/LF swallowed by a P/S run's [\r\n]* tail; digit index in its run; CR/LF ahead in the whitespace
    # run; ASCII letter inside a "punct + ASCII letters" token
    sw, ds, hna, a_in, cnt = [False] * n, [False] * n, [False] * n, [False] * n, 0
    for i in range(n):
        if nl[i]:
            j = i - 1
            while j >= 0 and nl[j]:
                j -= 1
            sw[i] = j >= 0 and k[j] == PS
        if k[i] == NUM:
            ds[i] = cnt % 3 == 0
            cnt += 1
        else:
            cnt = 0
        if k[i] == WSP and not nl[i]:
            j = i + 1
            while j < n and k[j] == WSP:
                if nl[j]:
                    hna[i] = True
                    break
                j += 1
        if aalpha(c[i]):
            j = i - 1
            while j >= 0 and aalpha(c[j]):
                j -= 1
            a_in[i] = j >= 0 and a_start[j]
    out = []
    for i in range(n):
        b = k[i]
        if i == 0:
            st = True
        else:
            a = k[i - 1]
            if b == NUM:
                st = ds[i]
            elif b == CJK:
                st = a != CJK
            elif a in (NUM, CJK):
                st = True                                   # a new piece
            elif b == LET:
                if a == LET:
                    st = a_in[i - 1] and not aalpha(c[i])   # "punct + ASCII letters" ends at the first other letter
                elif a == PS:
                    st = not (a_start[i - 1] and aalpha(c[i]))
                elif a == WSP:
                    st = nl[i - 1]                          # any other whitespace char is the letters' prefix
                else:
                    st = False                              # OTH: the letters' prefix
            elif b == PS:
                st = ps_start(i)
            elif b == OTH:
                st = a != OTH or (i + 1 < n and k[i + 1] == LET)
            elif nl[i]:
                st = (not sw[i]) and a != WSP
            elif hna[i]:
                st = a != WSP or (nl[i - 1] and sw[i - 1])
            else:
                nxt_open = i + 1 < n and k[i + 1] not in (WSP, NUM, CJK)   # a non-space char of the SAME piece follows
                st = a != WSP or nl[i - 1] or nxt_open
        if st:
            out.append(i)
    return out


ALPHA3 = list("ab  \t\n\r''.!12Z") + ["é", "日", "ひ", "カ", "́", "\x01", " ", "　", "\n\n", "!\n", " \n", "$", "€", "。",
                                     "²", "٣", ".com", " !", "\x7f", "ß", "!a", ".é", "\x01a"]


def test_deepseek_v3_rules_equal_the_sequential_scan():
    rnd = random.Random(9)
    for _ in range(150000):
        s = "".join(rnd.choice(ALPHA3) for _ in range(rnd.randrange(0, 14)))
        assert seq3(s) == rules3(s), repr(s)
