"""Logical query model + a small SQL front-end (tooling).

The reference compiles SQL to a `QueryContext` with Calcite (pinot-common, out of scope for this
build: SURVEY.md §2b "run unchanged before the hot path").  Tests and the benchmark need the same
starting point, so this module parses the SQL subset the hot path covers

    SELECT <agg | ident>, ... FROM <table> [WHERE <bool-expr>] [GROUP BY ident, ...] [LIMIT n]
    agg   := (COUNT(*) | SUM|MIN|MAX|AVG|DISTINCTCOUNT(ident)) [FILTER(WHERE <bool-expr>)]
    pred  := ident (=|!=|<>|<|<=|>|>=) literal | ident [NOT] IN (lit, ...) | ident BETWEEN lit AND lit
           | ident IS [NOT] NULL

into the logical `QueryContext` below (predicate literals are still strings, as in Pinot's
`Predicate` classes: pinot-common/.../request/context/predicate/*.java).  Lowering to dictIds and
index selection is NOT done here — that is the executor's host layer (and, independently, the oracle).
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from enum import IntEnum
from typing import Dict, List, Optional, Union


class PredicateType(IntEnum):
    EQ = 0
    NOT_EQ = 1
    IN = 2
    NOT_IN = 3
    RANGE = 4
    IS_NULL = 5          # BitmapBasedFilterOperator over the null-value vector; EmptyFilterOperator without one (FilterPlanNode.java:294-300)
    IS_NOT_NULL = 6      # ... exclusive; MatchAllFilterOperator without one (FilterPlanNode.java:301-307)


class AggOp(IntEnum):
    COUNT = 0
    SUM = 1
    MIN = 2
    MAX = 3
    AVG = 4
    DISTINCTCOUNT = 5


@dataclass
class Predicate:
    type: PredicateType
    column: str
    values: List[str] = field(default_factory=list)   # EQ/NEQ: 1 value, IN/NOT_IN: n
    lower: Optional[str] = None                       # RANGE; None = unbounded
    upper: Optional[str] = None
    lower_inclusive: bool = False
    upper_inclusive: bool = False


@dataclass
class And:
    children: List["FilterNode"]


@dataclass
class Or:
    children: List["FilterNode"]


@dataclass
class Not:
    child: "FilterNode"


FilterNode = Union[And, Or, Not, Predicate]


@dataclass
class Aggregation:
    op: AggOp
    column: Optional[str]        # None for COUNT(*)
    filter: Optional["FilterNode"] = None    # AGG(...) FILTER(WHERE ...): QueryContext.getFilteredAggregationFunctions()

    def __str__(self):
        return f"{self.op.name.lower()}({self.column or '*'})"


def postfix_of(flt: Optional["FilterNode"]):
    """[(kind, n_children, predicate_index)], [Predicate] — AND=0 OR=1 NOT=2 PRED=3."""
    nodes, preds = [], []

    def walk(n):
        if isinstance(n, Predicate):
            preds.append(n)
            nodes.append((3, 0, len(preds) - 1))
        elif isinstance(n, Not):
            walk(n.child)
            nodes.append((2, 1, -1))
        else:
            for c in n.children:
                walk(c)
            nodes.append((0 if isinstance(n, And) else 1, len(n.children), -1))

    if flt is not None:
        walk(flt)
    return nodes, preds


@dataclass
class QueryContext:
    """The slice of CTR/query/request/context/QueryContext.java the hot path reads."""
    table: str
    aggregations: List[Aggregation]
    group_by: List[str] = field(default_factory=list)
    filter: Optional[FilterNode] = None
    # InstancePlanMakerImplV2.java:70-97 defaults
    num_groups_limit: int = 100_000
    max_initial_result_holder_capacity: int = 10_000
    skip_indexes: Dict[str, List[str]] = field(default_factory=dict)   # column -> ["inverted", ...]
    skip_inverted_all: bool = False
    limit: int = 10
    # ORDER BY expressions that name a group-by column (kind 0, index into group_by) or an aggregation of the SELECT list
    # (kind 1, index into aggregations): [(kind, index, descending)]
    order_by: List[tuple] = field(default_factory=list)
    # CommonConstants.Server defaults: DEFAULT_MIN_SERVER_GROUP_TRIM_SIZE 5000, DEFAULT_MIN_SEGMENT_GROUP_TRIM_SIZE -1,
    # DEFAULT_GROUPBY_TRIM_THRESHOLD 1_000_000 (query options minServerGroupTrimSize / minSegmentGroupTrimSize / groupTrimThreshold)
    min_server_group_trim_size: int = 5000
    min_segment_group_trim_size: int = -1
    group_trim_threshold: int = 1_000_000
    # query option enableNullHandling (QueryContext.isNullHandlingEnabled): three-valued filters, aggregations skip null inputs
    null_handling: bool = False

    def trim(self, combined: bool):
        """(trim_size, trim_threshold) the combine layer (combined) or the segment operator would apply: GroupByUtils.
        getTableCapacity = max(5 x LIMIT, min trim size); (0, 0) when there is no ORDER BY or trimming is disabled."""
        m = self.min_server_group_trim_size if combined else self.min_segment_group_trim_size
        if not self.order_by or not self.group_by or m <= 0:
            return 0, 0
        size = max(min(5 * self.limit, 2**31 - 1), m)
        thr = self.group_trim_threshold if combined else size     # (the segment-level trim has no threshold: GroupByOperator trims whenever it holds more)
        if combined and (thr <= 0 or thr > 1_000_000_000):
            return 0, 0
        return size, max(thr, 2 * size) if combined else size

    def filter_postfix(self):
        """[(kind, n_children, predicate_index)], [Predicate] — AND=0 OR=1 NOT=2 PRED=3."""
        return postfix_of(self.filter)

    def agg_filters(self):
        """Distinct aggregation filters (equal filter expressions share a swim-lane, AggregationFunctionUtils.java:333-366)
        and, per aggregation, the index of its filter (-1 = not filtered)."""
        filters, index = [], []
        for a in self.aggregations:
            if a.filter is None:
                index.append(-1)
                continue
            for i, f in enumerate(filters):
                if f == a.filter:
                    index.append(i)
                    break
            else:
                filters.append(a.filter)
                index.append(len(filters) - 1)
        return filters, index


# --------------------------------------------------------------------------- SQL subset parser

_TOKEN = re.compile(r"\s*(?:(?P<num>-?\d+\.\d*(?:[eE][-+]?\d+)?|-?\.\d+|-?\d+(?:[eE][-+]?\d+)?)"
                    r"|(?P<str>'(?:[^']|'')*')|(?P<id>[A-Za-z_][A-Za-z_0-9$]*|\"[^\"]+\")"
                    r"|(?P<op><=|>=|<>|!=|=|<|>|\(|\)|,|\*|;))")


def _tokenize(sql: str):
    pos, out = 0, []
    sql = sql.strip().rstrip(";")
    while pos < len(sql):
        m = _TOKEN.match(sql, pos)
        if not m:
            raise ValueError(f"cannot tokenize at: {sql[pos:pos + 20]!r}")
        pos = m.end()
        if m.group("num") is not None:
            out.append(("num", m.group("num")))
        elif m.group("str") is not None:
            out.append(("str", m.group("str")[1:-1].replace("''", "'")))
        elif m.group("id") is not None:
            t = m.group("id")
            out.append(("id", t[1:-1] if t.startswith('"') else t))
        else:
            out.append(("op", m.group("op")))
    return out


class _Parser:
    def __init__(self, toks):
        self.t = toks
        self.i = 0

    def peek(self, k=0):
        return self.t[self.i + k] if self.i + k < len(self.t) else (None, None)

    def kw(self, word):
        k, v = self.peek()
        return k == "id" and v.upper() == word

    def eat_kw(self, word):
        if not self.kw(word):
            raise ValueError(f"expected {word}, got {self.peek()}")
        self.i += 1

    def eat_op(self, op):
        k, v = self.peek()
        if k != "op" or v != op:
            raise ValueError(f"expected {op!r}, got {self.peek()}")
        self.i += 1

    def literal(self) -> str:
        k, v = self.peek()
        if k not in ("num", "str"):
            raise ValueError(f"expected literal, got {self.peek()}")
        self.i += 1
        return v

    def ident(self) -> str:
        k, v = self.peek()
        if k != "id":
            raise ValueError(f"expected identifier, got {self.peek()}")
        self.i += 1
        return v

    # bool-expr := or-expr
    def or_expr(self):
        kids = [self.and_expr()]
        while self.kw("OR"):
            self.i += 1
            kids.append(self.and_expr())
        return kids[0] if len(kids) == 1 else Or(kids)

    def and_expr(self):
        kids = [self.not_expr()]
        while self.kw("AND"):
            self.i += 1
            kids.append(self.not_expr())
        return kids[0] if len(kids) == 1 else And(kids)

    def not_expr(self):
        if self.kw("NOT"):
            self.i += 1
            return Not(self.not_expr())
        k, v = self.peek()
        if k == "op" and v == "(":
            self.i += 1
            e = self.or_expr()
            self.eat_op(")")
            return e
        return self.predicate()

    def predicate(self):
        col = self.ident()
        if self.kw("BETWEEN"):
            self.i += 1
            lo = self.literal()
            self.eat_kw("AND")
            hi = self.literal()
            return Predicate(PredicateType.RANGE, col, lower=lo, upper=hi, lower_inclusive=True, upper_inclusive=True)
        if self.kw("IS"):
            self.i += 1
            neg = False
            if self.kw("NOT"):
                self.i += 1
                neg = True
            self.eat_kw("NULL")
            return Predicate(PredicateType.IS_NOT_NULL if neg else PredicateType.IS_NULL, col)
        negate = False
        if self.kw("NOT"):
            self.i += 1
            negate = True
        if self.kw("IN"):
            self.i += 1
            self.eat_op("(")
            vals = [self.literal()]
            while self.peek() == ("op", ","):
                self.i += 1
                vals.append(self.literal())
            self.eat_op(")")
            return Predicate(PredicateType.NOT_IN if negate else PredicateType.IN, col, values=vals)
        if negate:
            raise ValueError("NOT must be followed by IN here")
        k, op = self.peek()
        if k != "op":
            raise ValueError(f"expected comparison operator, got {self.peek()}")
        self.i += 1
        v = self.literal()
        if op == "=":
            return Predicate(PredicateType.EQ, col, values=[v])
        if op in ("!=", "<>"):
            return Predicate(PredicateType.NOT_EQ, col, values=[v])
        if op == "<":
            return Predicate(PredicateType.RANGE, col, upper=v, upper_inclusive=False)
        if op == "<=":
            return Predicate(PredicateType.RANGE, col, upper=v, upper_inclusive=True)
        if op == ">":
            return Predicate(PredicateType.RANGE, col, lower=v, lower_inclusive=False)
        if op == ">=":
            return Predicate(PredicateType.RANGE, col, lower=v, lower_inclusive=True)
        raise ValueError(f"unsupported operator {op}")


_AGGS = {"COUNT": AggOp.COUNT, "SUM": AggOp.SUM, "MIN": AggOp.MIN, "MAX": AggOp.MAX, "AVG": AggOp.AVG,
         "DISTINCTCOUNT": AggOp.DISTINCTCOUNT}


def parse_sql(sql: str) -> QueryContext:
    p = _Parser(_tokenize(sql))
    options = {}
    while p.kw("SET"):
        p.i += 1
        k = p.ident()
        p.eat_op("=")
        if p.peek()[0] == "id":           # SET enableNullHandling = true
            options[k.lower()] = p.peek()[1]
            p.i += 1
        else:
            options[k.lower()] = p.literal()
        if p.peek() == ("op", ";"):
            p.i += 1
    p.eat_kw("SELECT")
    aggs: List[Aggregation] = []
    select_idents: List[str] = []
    while True:
        name = p.ident()
        if p.peek() == ("op", "("):
            p.i += 1
            op = _AGGS.get(name.upper())
            if op is None:
                raise ValueError(f"unsupported aggregation function {name}")
            if p.peek() == ("op", "*"):
                p.i += 1
                col = None
            else:
                col = p.ident()
            p.eat_op(")")
            agg_filter = None
            if p.kw("FILTER"):
                p.i += 1
                p.eat_op("(")
                p.eat_kw("WHERE")
                agg_filter = p.or_expr()
                p.eat_op(")")
            aggs.append(Aggregation(op, col, agg_filter))
        else:
            select_idents.append(name)
        if p.peek() == ("op", ","):
            p.i += 1
            continue
        break
    p.eat_kw("FROM")
    table = p.ident()
    flt = None
    if p.kw("WHERE"):
        p.i += 1
        flt = p.or_expr()
    group_by: List[str] = []
    if p.kw("GROUP"):
        p.i += 1
        p.eat_kw("BY")
        group_by.append(p.ident())
        while p.peek() == ("op", ","):
            p.i += 1
            group_by.append(p.ident())
    order_by = []
    if p.kw("ORDER"):
        p.i += 1
        p.eat_kw("BY")
        while True:
            name = p.ident()
            if p.peek() == ("op", "("):
                p.i += 1
                op = _AGGS.get(name.upper())
                if p.peek() == ("op", "*"):
                    p.i += 1
                    col = None
                else:
                    col = p.ident()
                p.eat_op(")")
                ob_filter = None
                if p.kw("FILTER"):          # names the SELECT-list entry with the identical FILTER clause
                    p.i += 1
                    p.eat_op("(")
                    p.eat_kw("WHERE")
                    ob_filter = p.or_expr()
                    p.eat_op(")")
                hits = [i for i, a in enumerate(aggs) if a.op == op and a.column == col and a.filter == ob_filter]
                if not hits:
                    raise ValueError(f"ORDER BY {name}({col or '*'}){' FILTER(...)' if ob_filter is not None else ''} is not in the SELECT list")
                ob = (1, hits[0])
            else:
                if name not in group_by:
                    raise ValueError(f"ORDER BY {name} is not a group-by column")
                ob = (0, group_by.index(name))
            desc = False
            if p.kw("DESC"):
                p.i += 1
                desc = True
            elif p.kw("ASC"):
                p.i += 1
            order_by.append((ob[0], ob[1], desc))
            if p.peek() == ("op", ","):
                p.i += 1
                continue
            break
    limit = 10
    if p.kw("LIMIT"):
        p.i += 1
        limit = int(p.literal())
    if p.i != len(p.t):
        raise ValueError(f"trailing tokens: {p.t[p.i:]}")
    if not aggs:
        raise ValueError("only aggregation / group-by queries are on this path")
    q = QueryContext(table=table, aggregations=aggs, group_by=group_by, filter=flt, limit=limit, order_by=order_by)
    for opt, attr in (("minservergrouptrimsize", "min_server_group_trim_size"), ("minsegmentgrouptrimsize", "min_segment_group_trim_size"),
                      ("grouptrimthreshold", "group_trim_threshold")):
        if opt in options:
            setattr(q, attr, int(options[opt]))
    q.null_handling = str(options.get("enablenullhandling", "false")).lower() == "true"
    if "numgroupslimit" in options:
        q.num_groups_limit = int(options["numgroupslimit"])
    if "maxinitialresultholdercapacity" in options:
        q.max_initial_result_holder_capacity = int(options["maxinitialresultholdercapacity"])
    if options.get("filteredaggregationsskipemptygroups", "false").lower() == "true":
        raise ValueError("filteredAggregationsSkipEmptyGroups is not offloaded (the plan maker declines)")
    if "skipindexes" in options:     # e.g. 'c1=inverted,c2=inverted'
        for part in options["skipindexes"].split(","):
            if "=" in part:
                c, kinds = part.split("=", 1)
                q.skip_indexes[c.strip()] = [k.strip().lower() for k in kinds.split("|")]
    return q
