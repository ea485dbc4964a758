"""Tiny SQL front-end for tests: turns the reference's own test query strings (Tests/ExecuteTest.cpp) into the
RelAlgExecutionUnit mirror, for the subset of the path:

    SELECT <col | COUNT(*) | COUNT(c) | SUM(c) | MIN(c) | MAX(c) | AVG(c)>, ...
    FROM <table> [[LEFT] JOIN <inner> ON <table>.<c> = <inner>.<c>] [WHERE <c OP literal | c IS [NOT] NULL | c [NOT] IN (l, ...) | c BETWEEN l AND l | NOT <factor>>
                  {AND|OR} ... with parentheses] [GROUP BY c {, c}]
    [ORDER BY <position | target text | target alias> [ASC|DESC] [NULLS FIRST|LAST] {, ...}] [LIMIT n] [OFFSET m]

It plays the role Calcite + RelAlgTranslator play in the reference (kept, out of scope) and is test infrastructure.
Like RelAlgTranslator/QualsConjunctiveForm, a top-level AND is split into separate quals, and a `col OP const`
conjunct is a "simple qual" (Analyzer::BinOper::normalize_simple_predicate, QueryEngine/RelAlgExecutor.cpp
translation of filters: simple_quals vs quals).
"""
from __future__ import annotations

import re
from typing import List, Tuple

from heavydb_b200 import abi

_TOK = re.compile(r"\s*('(?:[^']|'')*'|<>|<=|>=|!=|[(),*<>=]|[A-Za-z_][A-Za-z_0-9]*(?:\.[A-Za-z_][A-Za-z_0-9]*)?|-?\d+\.\d*(?:[eE][-+]?\d+)?|-?\d+)")
_OPS = {"=": abi.kEQ, "<>": abi.kNE, "!=": abi.kNE, "<": abi.kLT, ">": abi.kGT, "<=": abi.kLE, ">=": abi.kGE}
_AGGS = {"COUNT": abi.kCOUNT, "SUM": abi.kSUM, "MIN": abi.kMIN, "MAX": abi.kMAX, "AVG": abi.kAVG}


def _tokens(s: str) -> List[str]:
    s = s.strip().rstrip(";")
    out, pos = [], 0
    while pos < len(s):
        m = _TOK.match(s, pos)
        if not m:
            raise ValueError(f"cannot tokenize at: {s[pos:]!r}")
        out.append(m.group(1))
        pos = m.end()
    return out


class _P:
    def __init__(self, toks, table: abi.Table, names: List[str], bigint_count: bool, inner=None, dicts=None):
        self.t, self.i = toks, 0
        self.dicts = {k.lower(): v for k, v in (dicts or {}).items()}   # column name -> strings in dictionary-id order
        self.b = abi.UnitBuilder(table)
        self.names = [n.lower() for n in names]
        self.bigint_count = bigint_count
        # one INNER join level: inner = (abi.Table, [column names]); set before any column is resolved
        self.inner_names = [n.lower() for n in inner[1]] if inner else []
        self.outer_alias = self.inner_alias = None
        if inner:
            self.b.inner = inner[0]

    def peek(self):
        return self.t[self.i] if self.i < len(self.t) else None

    def eat(self, expect=None):
        tok = self.peek()
        if tok is None or (expect is not None and tok.upper() != expect):
            raise ValueError(f"expected {expect}, got {tok}")
        self.i += 1
        return tok

    def colref(self, name):
        """(column id, rte_idx).  `alias.col` is resolved by alias, a bare name in the outer table first."""
        name = name.lower()
        if "." in name:
            alias, col = name.split(".", 1)
            if self.inner_alias is not None and alias == self.inner_alias:
                return self.inner_names.index(col), 1
            return self.names.index(col), 0
        if name in self.names:
            return self.names.index(name), 0
        return self.inner_names.index(name), 1

    def colid(self, name):
        c, rte = self.colref(name)
        assert rte == 0, f"{name}: inner-table column where only outer columns are supported"
        return c

    # cond := term {OR term}; term := factor {AND factor}; factor := '(' cond ')' | col OP literal
    def cond(self):
        e = self.term()
        while self.peek() and self.peek().upper() == "OR":
            self.eat()
            e = self.b.binop(abi.kOR, e, self.term())
        return e

    def term(self):
        e = self.factor()
        while self.peek() and self.peek().upper() == "AND":
            self.eat()
            e = self.b.binop(abi.kAND, e, self.factor())
        return e

    def literal_cmp(self, col, op, lit, rte=0):
        tbl = self.b.inner if rte else self.b.table
        if lit.startswith("'"):
            # a string literal against a dictionary-encoded column: the reference translates it to the column's dictionary id
            # (StringDictionaryProxy::getIdOfString; an unknown string is INVALID_STR_ID = -1, which no row holds) and compares ids
            # — for = and <> only; an ordering comparison needs the dictionary itself (CodeGenerator::codegenCmp -> string ops)
            name = (self.inner_names if rte else self.names)[col]
            if tbl.col_types[col][0] not in (abi.kTEXT, abi.kVARCHAR, abi.kCHAR) or name not in self.dicts:
                raise ValueError(f"string literal {lit} against a column without a dictionary")
            if op not in (abi.kEQ, abi.kNE):
                raise ValueError("string ordering comparisons need the dictionary: outside the path")
            text = lit[1:-1].replace("''", "'")
            sid = self.dicts[name].index(text) if text in self.dicts[name] else -1
            return self.b.cmp(col, op, sid, abi.kBIGINT, rte)
        if tbl.col_types[col][0] in abi.DECIMAL_TYPES:
            # the analyzer folds the literal to the common DECIMAL type: same scale as the column when the literal has no
            # more fraction digits than the column (Constant::do_cast); otherwise the COLUMN would be cast — not this path
            import decimal
            scale = tbl.col_scales.get(col, 0)
            v = decimal.Decimal(lit).scaleb(scale)
            if v != v.to_integral_value():
                raise ValueError(f"literal {lit} has more fraction digits than DECIMAL scale {scale}")
            return self.b.cmp(col, op, int(v), tbl.col_types[col][0], rte, scale=scale)
        if tbl.col_types[col][0] == abi.kFLOAT:
            # common_numeric_type(FLOAT, <int / decimal literal>) = FLOAT: the literal is folded to a FLOAT Datum
            return self.b.cmp(col, op, float(lit), abi.kFLOAT, rte)
        if re.fullmatch(r"-?\d+", lit):
            return self.b.cmp(col, op, int(lit), abi.kBIGINT, rte)
        return self.b.cmp(col, op, float(lit), abi.kDOUBLE, rte)

    def factor(self):
        if self.peek() == "(":
            self.eat()
            e = self.cond()
            self.eat(")")
            return e
        if self.peek().upper() == "NOT":          # Analyzer::UOper(kNOT, ...)
            self.eat()
            return self.b.uoper(abi.kNOT, self.factor())
        col, rte = self.colref(self.eat())
        nxt = self.peek().upper()
        if nxt == "IS":                            # c IS NULL -> UOper(kISNULL, c); IS NOT NULL -> NOT(ISNULL), like RelAlgTranslator
            self.eat()
            neg = self.peek().upper() == "NOT"
            if neg:
                self.eat()
            self.eat("NULL")
            e = self.b.uoper(abi.kISNULL, self.b.col(col, rte))
            return self.b.uoper(abi.kNOT, e) if neg else e
        neg = False
        if nxt == "NOT":
            self.eat()
            neg = True
            nxt = self.peek().upper()
        if nxt == "IN":                            # c IN (a, b, ...) -> OR of equalities (InValues codegen for short lists)
            self.eat()
            self.eat("(")
            e = self.literal_cmp(col, abi.kEQ, self.eat(), rte)
            while self.peek() == ",":
                self.eat()
                e = self.b.binop(abi.kOR, e, self.literal_cmp(col, abi.kEQ, self.eat(), rte))
            self.eat(")")
            return self.b.uoper(abi.kNOT, e) if neg else e
        if nxt == "BETWEEN":                       # Calcite expands BETWEEN to >= AND <=
            self.eat()
            lo = self.eat()
            self.eat("AND")
            hi = self.eat()
            e = self.b.binop(abi.kAND, self.literal_cmp(col, abi.kGE, lo, rte), self.literal_cmp(col, abi.kLE, hi, rte))
            return self.b.uoper(abi.kNOT, e) if neg else e
        op = _OPS[self.eat()]
        rhs = self.eat()
        if re.fullmatch(r"[A-Za-z_][A-Za-z_0-9.]*", rhs):     # column OP column
            c2, rte2 = self.colref(rhs)
            if self.dicts:   # ids of two dictionaries are not comparable: what the bridge's on_path() checks with getStringDictKey()
                n1 = (self.inner_names if rte else self.names)[col]
                n2 = (self.inner_names if rte2 else self.names)[c2]
                if n1 in self.dicts and n2 in self.dicts and self.dicts[n1] is not self.dicts[n2]:
                    raise ValueError(f"{n1} and {n2} use different dictionaries: string comparison, outside the path")
            return self.b.binop(op, self.b.col(col, rte), self.b.col(c2, rte2))
        return self.literal_cmp(col, op, rhs, rte)

    def target_text(self):
        """Canonical text of the target expression starting at the cursor (does not build nodes)."""
        j = self.i
        tok = self.t[j]
        if tok.upper() in _AGGS and j + 1 < len(self.t) and self.t[j + 1] == "(":
            k = self.t.index(")", j)
            return "".join(self.t[j:k + 1]).upper(), k + 1
        return tok.upper(), j + 1

    def target(self):
        tok = self.eat()
        if tok.upper() in _AGGS and self.peek() == "(":
            self.eat("(")
            if self.peek() == "*":
                self.eat()
                self.eat(")")
                return self.b.agg(abi.kCOUNT, None, self.bigint_count)
            distinct = False
            if self.peek().upper() == "DISTINCT":
                self.eat()
                distinct = True
            col, rte = self.colref(self.eat())
            self.eat(")")
            return self.b.agg(_AGGS[tok.upper()], col, self.bigint_count, rte, is_distinct=distinct)
        return self.b.col(*self.colref(tok))


def _conjuncts(b: abi.UnitBuilder, e: int) -> List[int]:
    n = b.nodes[e]
    if n.kind == abi.EXPR_BIN_OPER and n.op == abi.kAND:
        return _conjuncts(b, n.left) + _conjuncts(b, n.right)
    return [e]


def parse(sql: str, table: abi.Table, names: List[str], bigint_count: bool = False, inner=None, dicts=None) -> abi.BuiltUnit:
    """inner = (abi.Table, [names]) of the table named after JOIN (one concatenated fragment); dicts = {column: [strings in id
    order]} for string literals against dictionary-encoded columns."""
    toks = _tokens(sql)
    p = _P(toks, table, names, bigint_count, inner, dicts)
    ups = [t.upper() for t in toks]
    fi = ups.index("FROM")
    p.outer_alias = toks[fi + 1].lower()
    ji = fi + 2
    if ji < len(toks) and ups[ji] == "LEFT":
        p.b.join_type = 1          # known before any column of the inner table is resolved (they become nullable)
        ji += 1
    if ji < len(toks) and ups[ji] == "JOIN":
        assert inner is not None, "JOIN needs the inner table"
        p.inner_alias = toks[ji + 1].lower()
    p.eat("SELECT")
    texts, targets, aliases = [], [], {}

    def one_target():
        texts.append(p.target_text()[0])
        targets.append(p.target())
        if p.peek() and p.peek().upper() == "AS":     # <target> AS alias — usable in ORDER BY
            p.eat()
            aliases[p.eat().upper()] = len(targets)
        elif p.peek() and p.peek() != "," and p.peek().upper() != "FROM" and re.fullmatch(r"[A-Za-z_][A-Za-z_0-9]*", p.peek()):
            aliases[p.eat().upper()] = len(targets)

    one_target()
    while p.peek() == ",":
        p.eat()
        one_target()
    p.eat("FROM")
    p.eat()  # table name
    if p.peek() and p.peek().upper() == "LEFT":
        p.eat()
    if p.peek() and p.peek().upper() == "JOIN":   # join_quals[0] = {a = b}, INNER or LEFT
        p.eat()
        p.eat()  # inner table name
        p.eat("ON")
        (c1, r1), _, (c2, r2) = p.colref(p.eat()), p.eat("="), p.colref(p.eat())
        assert {r1, r2} == {0, 1}, "ON must compare an outer with an inner column"
        p.b.join(inner[0], c1 if r1 == 0 else c2, c2 if r1 == 0 else c1, p.b.join_type)
    if p.peek() and p.peek().upper() == "WHERE":
        p.eat()
        e = p.cond()
        for c in _conjuncts(p.b, e):
            n = p.b.nodes[c]
            simple = n.kind == abi.EXPR_BIN_OPER and n.op not in (abi.kAND, abi.kOR)
            if simple and p.b.nodes[n.right].kind != abi.EXPR_CONSTANT:
                simple = False          # column OP column is never a simple qual
            if simple:
                # an integer column against an fp literal is `CAST(col AS DOUBLE) OP lit` in the reference; only
                # int->int / timestamp casts survive BinOper::normalize_simple_predicate, so it is NOT a simple qual
                col_fp = p.b.nodes[n.left].type in (abi.kDOUBLE, abi.kFLOAT)
                lit_fp = p.b.nodes[n.right].type in (abi.kDOUBLE, abi.kFLOAT)
                simple = col_fp == lit_fp
            p.b.add_qual(c, simple=simple)
    if p.peek() and p.peek().upper() == "GROUP":
        p.eat()
        p.eat("BY")
        p.b.group_by(*p.colref(p.eat()))
        while p.peek() == ",":
            p.eat()
            p.b.group_by(*p.colref(p.eat()))
    if p.peek() and p.peek().upper() == "ORDER":
        p.eat()
        p.eat("BY")
        while True:
            if re.fullmatch(r"\d+", p.peek()):
                tle = int(p.eat())
            elif p.peek().upper() in aliases:
                tle = aliases[p.eat().upper()]
            else:
                text, nxt = p.target_text()
                p.i = nxt
                tle = texts.index(text) + 1
            desc, nulls_first = False, None
            if p.peek() and p.peek().upper() in ("ASC", "DESC"):
                desc = p.eat().upper() == "DESC"
            if p.peek() and p.peek().upper() == "NULLS":
                p.eat()
                nulls_first = p.eat().upper() == "FIRST"
            p.b.order_by(tle, desc, nulls_first)
            if p.peek() != ",":
                break
            p.eat()
    if p.peek() and p.peek().upper() == "LIMIT":
        p.eat()
        p.b.limit = int(p.eat())
    if p.peek() and p.peek().upper() == "OFFSET":
        p.eat()
        p.b.offset = int(p.eat())
    if p.peek() is not None:
        raise ValueError(f"trailing tokens: {p.t[p.i:]}")
    for t in targets:
        p.b.target(t)
    # get_scan_limit (RelAlgExecutor.cpp:3442-3449, :3630-3632): LIMIT without ORDER BY over a non-aggregate source scans at
    # most limit + offset rows; aggregate units keep scan_limit 0
    aggregate = p.b.groupby or any(p.b.nodes[t].kind == abi.EXPR_AGG for t in targets)
    if not aggregate and p.b.estimator_kind == 0 and not p.b.order and p.b.limit is not None:
        p.b.scan_limit = p.b.limit + p.b.offset
    return p.b.build()


# ---- work units of a multi-step query ------------------------------------------------------------------------------------
_CLAUSES = ("FROM", "WHERE", "GROUP", "HAVING", "ORDER", "LIMIT", "OFFSET")
_KEYWORDS = set(_CLAUSES) | {"SELECT", "JOIN", "LEFT", "INNER", "ON", "AS", "BY"}


class Step:
    """One work unit of parse_steps: `sql` is a query parse() accepts over its input tables.  `source` / `inner` name them:
    a base table name (a str) or the index of an earlier step whose result is read as a temporary table; `inner` is None
    without a join.  `names` are the step's output column names (the temporary table's column names)."""

    def __init__(self, sql: str, source, inner, names: List[str]):
        self.sql, self.source, self.inner, self.names = sql, source, inner, names

    def __repr__(self):
        return f"Step({self.sql!r}, source={self.source!r}, inner={self.inner!r}, names={self.names})"


def _split_clauses(toks: List[str]):
    """{clause: tokens} of one SELECT, split at parenthesis depth 0 (GROUP / ORDER without their BY)."""
    out, cur, depth = {"SELECT": []}, "SELECT", 0
    for i, tok in enumerate(toks[1:], 1):
        up = tok.upper()
        if depth == 0 and up in _CLAUSES:
            cur = up
            out[cur] = []
            continue
        if depth == 0 and up == "BY" and cur in ("GROUP", "ORDER") and not out[cur]:
            continue
        depth += tok == "("
        depth -= tok == ")"
        out[cur].append(tok)
    return out


def _split_commas(toks: List[str]) -> List[List[str]]:
    parts, cur, depth = [], [], 0
    for tok in toks:
        if tok == "," and depth == 0:
            parts.append(cur)
            cur = []
            continue
        depth += tok == "("
        depth -= tok == ")"
        cur.append(tok)
    return parts + [cur] if cur else parts


def _is_agg(toks: List[str], j: int) -> bool:
    return toks[j].upper() in _AGGS and j + 1 < len(toks) and toks[j + 1] == "("


def _agg_text(toks: List[str], j: int):
    """(canonical text, index after) of the aggregate call at toks[j] — the text parse()'s ORDER BY matching uses."""
    k = toks.index(")", j)
    return "".join(toks[j:k + 1]).upper(), k + 1


def _output_names(select: List[List[str]]) -> List[str]:
    """Column names of a SELECT list: the alias, else a column's own name, else EXPR<i> (Calcite's EXPR$<i>)."""
    names = []
    for i, t in enumerate(select):
        if len(t) >= 2 and re.fullmatch(r"[A-Za-z_][A-Za-z_0-9]*", t[-1]) and (t[-2].upper() == "AS" or t[-2] == ")" or len(t) == 2):
            names.append(t[-1].lower())
        elif len(t) == 1:
            names.append(t[0].split(".")[-1].lower())
        else:
            names.append(f"expr{i}")
    return names


def _source(toks: List[str], j: int, steps: List[Step], tables):
    """A FROM item at toks[j]: a table name or a parenthesised SELECT, then an optional [AS] alias.  Returns (source, the
    name the step's SQL uses for it, its column names, index after)."""
    if toks[j] == "(":
        depth, k = 0, j
        while True:
            depth += toks[k] == "("
            depth -= toks[k] == ")"
            if depth == 0:
                break
            k += 1
        src = _plan(toks[j + 1:k], steps, tables)
        j = k + 1
        default = f"tmp{src}"
        names = steps[src].names
    else:
        src = toks[j].lower()
        default = src
        names = tables[src][1] if src in tables else None
        j += 1
    if j < len(toks) and toks[j].upper() == "AS":
        j += 1
    alias = None
    if j < len(toks) and toks[j].upper() not in _KEYWORDS and re.fullmatch(r"[A-Za-z_][A-Za-z_0-9]*", toks[j]):
        alias = toks[j].lower()
        j += 1
    return src, alias or default, names, j


def _plan(toks: List[str], steps: List[Step], tables) -> int:
    """Append the steps of one SELECT (its subqueries first) and return the index of the step that yields its rows."""
    if not toks or toks[0].upper() != "SELECT":
        raise ValueError("a step must be a SELECT")
    cl = _split_clauses(toks)
    frm = cl.get("FROM")
    if not frm:
        raise ValueError("SELECT without FROM")
    src, sname, _names, j = _source(frm, 0, steps, tables)
    from_sql, inner = [sname], None
    if j < len(frm):
        if frm[j].upper() == "LEFT":
            from_sql.append("LEFT")
            j += 1
        if frm[j].upper() == "INNER":
            j += 1
        if frm[j].upper() != "JOIN":
            raise ValueError(f"unexpected {frm[j]} in FROM")
        inner, iname, _inames, j = _source(frm, j + 1, steps, tables)
        from_sql += ["JOIN", iname] + frm[j:]
    select = _split_commas(cl["SELECT"])
    tail = []
    for c in ("WHERE", "GROUP", "HAVING", "ORDER", "LIMIT", "OFFSET"):
        if c in cl and c != "HAVING":
            tail += [c] + (["BY"] if c in ("GROUP", "ORDER") else []) + cl[c]
    if "HAVING" not in cl:
        names = _output_names(select)
        steps.append(Step(" ".join(["SELECT"] + cl["SELECT"] + ["FROM"] + from_sql + tail) + ";", src, inner, names))
        return len(steps) - 1
    # HAVING: an Aggregate followed by a Filter is two compounds (RelAlgDagBuilder).  Step 1 computes the GROUP BY keys and
    # every aggregate SELECT, HAVING or ORDER BY uses; step 2 projects the SELECT list out of it, filtered by the HAVING
    # condition over its columns, then sorts and limits.
    if "GROUP" not in cl:
        raise ValueError("HAVING without GROUP BY")
    keys = _split_commas(cl["GROUP"])
    if any(len(k) != 1 for k in keys):
        raise ValueError("GROUP BY expressions are outside this front-end")
    key_names = [k[0].split(".")[-1].lower() for k in keys]
    if len(set(key_names)) != len(key_names):
        raise ValueError("two GROUP BY keys of one name")
    aggs, agg_names = [], {}
    out_names = _output_names(select)
    for i, t in enumerate(select):
        if _is_agg(t, 0):
            text = _agg_text(t, 0)[0]
            if text not in agg_names:
                aggs.append(t[:t.index(")") + 1])
                agg_names[text] = out_names[i] if out_names[i] not in key_names and not out_names[i].startswith("expr") \
                    else f"agg{len(aggs) - 1}"
        elif len(t) != 1 and not (len(t) == 3 and t[1].upper() == "AS") and len(t) != 2:
            raise ValueError("expressions in the SELECT list are outside this front-end")
    for c in ("HAVING", "ORDER"):
        t = cl.get(c, [])
        for j2 in range(len(t)):
            if _is_agg(t, j2):
                text, k = _agg_text(t, j2)
                if text not in agg_names:
                    aggs.append(t[j2:k])
                    agg_names[text] = f"agg{len(aggs) - 1}"
    step1 = ["SELECT", ", ".join(keys_[0] for keys_ in keys)] + [", " + " ".join(a) for a in aggs]
    step1 = " ".join(step1).replace(" ,", ",")
    tail1 = []
    if "WHERE" in cl:
        tail1 += ["WHERE"] + cl["WHERE"]
    tail1 += ["GROUP", "BY"] + cl["GROUP"]
    steps.append(Step(" ".join([step1, "FROM"] + from_sql + tail1) + ";", src, inner, key_names + list(agg_names.values())))
    first = len(steps) - 1

    def rewrite(t: List[str]) -> List[str]:
        out, j2 = [], 0
        while j2 < len(t):
            if _is_agg(t, j2):
                text, j2 = _agg_text(t, j2)
                out.append(agg_names[text])
                continue
            tok = t[j2]
            if re.fullmatch(r"[A-Za-z_][A-Za-z_0-9]*\.[A-Za-z_][A-Za-z_0-9]*", tok):
                tok = tok.split(".")[-1]
            out.append(tok)
            j2 += 1
        return out

    proj = []
    for i, t in enumerate(select):
        col = agg_names[_agg_text(t, 0)[0]] if _is_agg(t, 0) else t[0].split(".")[-1].lower()
        proj.append(col if col == out_names[i] or out_names[i].startswith("expr") else f"{col} AS {out_names[i]}")
    tail2 = ["WHERE"] + rewrite(cl["HAVING"])
    if "ORDER" in cl:
        tail2 += ["ORDER", "BY"] + rewrite(cl["ORDER"])
    for c in ("LIMIT", "OFFSET"):
        if c in cl:
            tail2 += [c] + cl[c]
    names = [p.split(" AS ")[-1] for p in proj]
    steps.append(Step(" ".join(["SELECT", ", ".join(proj), "FROM", f"tmp{first}"] + tail2) + ";", first, None, names))
    return len(steps) - 1


def parse_steps(sql: str, table: abi.Table, names: List[str], tables=None) -> List[Step]:
    """The work units of `sql` in the order RelAlgDag makes them (an Aggregate followed by a Filter, a subquery in FROM
    and an aggregated subquery on the inner side of a join each end a unit), for queries over temporary tables:

        SELECT ... GROUP BY ... HAVING <cond> [ORDER BY ...] [LIMIT n] [OFFSET m]
        SELECT ... FROM (SELECT ...) [alias] ...                       (nested to any depth)
        SELECT ... FROM t [LEFT] JOIN (SELECT k, AGG(..) FROM d GROUP BY k) s ON t.a = s.k ...

    Each step is a query parse() accepts, over a base table or the result of an earlier step (read as a temporary table
    whose column names are that step's `names`).  `table` / `names` describe the table a FROM names when `tables`
    ({name: (abi.Table, [column names])}) does not list it; parse() itself is unchanged.  Raises ValueError for a shape
    outside this front-end."""
    toks = _tokens(sql)
    tables = {k.lower(): v for k, v in (tables or {}).items()}
    for tok_i, tok in enumerate(toks):
        up = tok.upper()
        if up == "FROM" and toks[tok_i + 1] != "(" and toks[tok_i + 1].lower() not in tables:
            tables[toks[tok_i + 1].lower()] = (table, list(names))
    steps: List[Step] = []
    _plan(toks, steps, tables)
    return steps
