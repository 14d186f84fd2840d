"""Matrix Market text exactly as sprs 0.7.1 `write_matrix_market` emits it for the reference
(vartrix src/main.rs:381-389; layout observed in every golden, SURVEY.md A.9):
header, `% written by sprs`, `rows cols nnz`, then `row+1 col+1 value` in insertion order with the
value printed like Rust's `{}` for f64 (shortest round-trip digits, never an exponent, `NaN`)."""
from __future__ import annotations

from decimal import Decimal


def fmt_f64(v: float) -> str:
    if v != v:
        return "NaN"
    if v == float("inf"):
        return "inf"
    if v == float("-inf"):
        return "-inf"
    if v == int(v) and abs(v) < 1e16:
        return str(int(v))
    return format(Decimal(repr(float(v))), "f")


def mtx_text(n_rows: int, n_cols: int, row, col, val) -> str:
    out = ["%%MatrixMarket matrix coordinate real general", "% written by sprs", f"{n_rows} {n_cols} {len(row)}"]
    out += [f"{int(r) + 1} {int(c) + 1} {fmt_f64(float(v))}" for r, c, v in zip(row, col, val)]
    return "\n".join(out) + "\n"


def write_mtx(path: str, n_rows: int, n_cols: int, row, col, val):
    with open(path, "w") as fh:
        fh.write(mtx_text(n_rows, n_cols, row, col, val))
