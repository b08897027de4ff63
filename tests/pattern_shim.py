"""TEST-ONLY numpy stand-in for quokka_b200.ops.pattern_search (csrc/pattern.cu), part of tests/cpu_shim.py, so that
OrderedStream.pattern_recognize runs through the planner, the executors and the gloo exchange without a GPU.

The search is the kernel's, row by row: the level scan (candidate bit, t > t(i-1), t <= t0 + maxspan, the link program), the
resume after the bound row, the end of a level no later program reads, the caps of the best match found so far and the step
budget.  tests/pattern_cases.py's brute-force enumeration is what it is checked against."""
from __future__ import annotations

import numpy as np
import torch

from quokka_b200 import _lib as L
from quokka_b200 import expr as E
from quokka_b200.ops import PatternBudgetError


def _link(prog, ev, r, cols, valid, vals):
    """fp64 postfix evaluation of one link program; None when it reads a NULL."""
    st = []
    for op, a0, a1, imm, _ in prog:
        if op == L.OP_COL:
            if a1 == ev:
                if valid[a0] is not None and not valid[a0][r]:
                    return None
                st.append(np.float64(cols[a0][r]))
            else:
                if vals[a1][a0] is None:
                    return None
                st.append(vals[a1][a0])
        elif op == L.OP_CONST:
            st.append(np.float64(imm))
        elif op == L.OP_NEG:
            st.append(-st.pop())
        elif op == L.OP_NOT:
            st.append(np.float64(st.pop() == 0.0))
        elif op == L.OP_SELECT:
            b, a, c = st.pop(), st.pop(), st.pop()
            st.append(a if c != 0.0 else b)
        else:
            b, a = st.pop(), st.pop()
            with np.errstate(all="ignore"):
                st.append({L.OP_ADD: lambda: a + b, L.OP_SUB: lambda: a - b, L.OP_MUL: lambda: a * b, L.OP_DIV: lambda: a / b,
                           L.OP_LT: lambda: np.float64(a < b), L.OP_LE: lambda: np.float64(a <= b), L.OP_GT: lambda: np.float64(a > b),
                           L.OP_GE: lambda: np.float64(a >= b), L.OP_EQ: lambda: np.float64(a == b), L.OP_NE: lambda: np.float64(a != b),
                           L.OP_AND: lambda: np.float64(a != 0.0 and b != 0.0), L.OP_OR: lambda: np.float64(a != 0.0 or b != 0.0)}[op]())
    return not st or st[0] != 0.0


def pattern_search(time, by, seg, n_by, cand, starts, m, maxspan, link_cols, link_valid, links, budget, rows_tested=None):
    """The argument checks of qk_pattern_search that the host can make, then its search."""
    if not 2 <= m <= L.PATTERN_MAX_EVENTS:
        raise L.QkError(f"qk_pattern_search: {m} events")
    if maxspan < 0 or budget < 1:
        raise L.QkError("qk_pattern_search: negative maxspan or budget < 1")
    if len(links) != m or links[0]:
        raise L.QkError("qk_pattern_search: bad link programs")
    for k, prog in enumerate(links):
        E.check_program(prog or [], f"pattern_search: link program {k}")
    if by.numel() != time.numel() or cand.numel() != time.numel() or seg.numel() != n_by + 1:
        raise L.QkError("pattern_search: inconsistent row counts or segment offsets")
    T, B, S, CAND = time.numpy(), by.numpy(), seg.numpy(), cand.numpy()
    cols = [c.numpy() for c in link_cols]
    valid = [None if v is None else v.numpy() for v in link_valid]
    read = 0
    for e, prog in enumerate(links):
        for op, a0, a1, *_ in prog or []:
            if op == L.OP_COL and a1 < e:
                read |= 1 << a1
    indep = [(not (read >> i) & 1) or i == m - 1 for i in range(m)]
    out = np.full((len(starts), m), -1, np.int32)
    over, first, total = 0, None, 0
    for si, s in enumerate(starts.numpy().tolist()):
        b = int(B[s]) if 0 <= s < len(T) else -1
        if not (0 <= b < n_by and S[b] <= s < S[b + 1] <= len(T)) or not CAND[s] & 1:
            continue
        end = int(S[b + 1])
        lim = int(T[s]) + int(maxspan)
        row, tb, pos = [0] * m, [0] * m, [0] * m
        vals = [[None] * len(cols) for _ in range(m)]

        def stage(e, r):
            vals[e] = [None if (valid[c] is not None and not valid[c][r]) else np.float64(cols[c][r]) for c in range(len(cols))]
        row[0], tb[0], pos[1] = s, int(T[s]), s + 1
        stage(0, s)
        best, brow = None, None
        tight = [True] * m
        tested, level = 0, 1
        while level >= 1:
            cap = min(lim, best[level]) if best is not None and tight[level] else lim
            found, p = -1, pos[level]
            while True:
                if p >= end or T[p] > cap:
                    break
                tested += 1
                if (CAND[p] >> level) & 1 and T[p] > tb[level - 1] and _link(links[level], level, p, cols, valid, vals):
                    found = p
                    break
                if tested > budget:
                    break
                p += 1
            if tested > budget:
                break
            if found >= 0:
                row[level], pos[level], tb[level] = found, found + 1, int(T[found])
                if level < m - 1:
                    stage(level, found)
                    tight[level + 1] = tight[level] and best is not None and tb[level] == best[level]
                    pos[level + 1] = found + 1
                    level += 1
                    continue
                best, brow = list(tb), list(row)
                tight = [True] * m
            level -= 1
            while level >= 1 and indep[level]:
                level -= 1
        total += tested
        if tested > budget:
            over += 1
            first = si if first is None else first
            continue
        if best is not None:
            out[si] = brow
    if rows_tested is not None:
        rows_tested += total
    if over:
        raise PatternBudgetError(f"pattern_search: {over} start(s) tested more than {budget} rows; the first is start {first}", first)
    return torch.from_numpy(out)
