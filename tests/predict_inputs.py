"""Seeded extractor output for the predict tests and tools/predict_rate.py: method lines `name ctx ctx ...` whose
contexts `token,path,token` cover what __main__.print_predictions has rules for (DESIGN.md §6i)."""
from __future__ import annotations

import numpy as np

# "Aa" and "BB" have the same Java String.hashCode (2112), and the literal numeric path "2112" has that key too
COLLIDING_PATHS = ["Aa", "BB", "2112", "AaAa", "BBBB", "AaBB", "BBAa"]
ODD_PATHS = ["", "-", "-5", "a|b", "(X)^(Y)"]


def node_paths(n: int, rng) -> list:
    """n path strings shaped like the extractor's: node types joined by ^ and _."""
    kinds = ["NameExpr", "MethodCallExpr", "BlockStmt", "IfStmt", "ReturnStmt", "VariableDeclarator", "FieldAccessExpr",
             "AssignExpr", "BinaryExpr", "Parameter", "ClassOrInterfaceType", "ExpressionStmt"]
    out = set()
    while len(out) < n:
        up = rng.integers(1, 5)
        down = rng.integers(1, 5)
        out.add("^".join("(%s)" % kinds[rng.integers(len(kinds))] for _ in range(up)) + "_" +
                "_".join("(%s)" % kinds[rng.integers(len(kinds))] for _ in range(down)))
    return sorted(out)


def synthetic_lines(n_methods: int, seed: int, tokens, names, max_bag: int = 230, n_paths: int = 500,
                    numeric_paths=(), zipf: float = 1.6, specials: bool = True) -> list:
    """n_methods method lines (str, without line ends).  Bags are Zipf-sized, capped at max_bag; with specials, some
    methods have no context, repeated contexts, colliding or odd paths, unknown tokens and doubled spaces, and some
    lines are blank or start with a space (skipped)."""
    rng = np.random.default_rng(seed)
    paths = node_paths(n_paths, rng) + list(numeric_paths)
    if specials:
        paths += COLLIDING_PATHS + ODD_PATHS
    tokens = list(tokens)
    lines = []
    for m in range(n_methods):
        bag = min(int(rng.zipf(zipf)), max_bag)
        if specials and m % 97 == 5:
            bag = 0                                                  # all padding: NaN attention and scores
        ctx = []
        for _ in range(bag):
            t1 = tokens[rng.integers(len(tokens))] if rng.random() > 0.05 else "unk%d" % rng.integers(1000)
            t2 = tokens[rng.integers(len(tokens))] if rng.random() > 0.05 else ""
            ctx.append("%s,%s,%s" % (t1, paths[int(rng.zipf(1.3)) % len(paths)], t2))
        if specials and bag > 2 and m % 7 == 0:
            ctx += ctx[:3]                                           # repeated triples, later values win
        line = " ".join([names[rng.integers(len(names))]] + ctx)
        if specials and m % 53 == 3:
            line = line.replace(" ", "  ", 2)                        # empty fields
        if specials and m % 61 == 7:
            line += " \x0b\x0c\x1c"                                  # trailing bytes rstrip removes
        lines.append(line)
        if specials and m % 89 == 11:
            lines.append("")                                         # skipped lines
            lines.append(" leading space skips the line,1,2")
    return lines
