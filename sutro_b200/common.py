"""Host helpers on the infer() path, mirroring the reference's argument handling
(`sutro/common.py:72-163`): column extraction, multi-column concatenation, schema
normalisation.  Same names, argument meaning and error behaviour; frames are
duck-typed (pandas always available, polars / pyarrow when installed).
"""
from __future__ import annotations

import math
import os
import sys
from typing import Any, Dict, List, Literal, Tuple, Type, Union

import pandas as pd

try:  # optional, exactly as a user of the reference would have it
    import polars as pl  # type: ignore
except Exception:  # pragma: no cover - polars is absent in this image
    pl = None

EmbeddingModelOptions = Literal["qwen-3-embedding-0.6b", "qwen-3-embedding-6b",
                                "qwen-3-embedding-8b"]
ModelOptions = Union[Literal["llama-3.1-8b", "qwen-3-4b", "qwen-3-14b", "qwen-3-14b-thinking",
                             "qwen-3-0.6b", "qwen-3-embedding-0.6b"],
                     str]


def is_jupyter() -> bool:
    return not sys.stdout.isatty()


def to_colored_text(text: Any, state: str = None) -> str:
    """Plain-text variant of the reference helper (sutro/common.py:166-193): colours are
    dropped whenever stdout is not a TTY there too."""
    return str(text)


def _is_polars_frame(data) -> bool:
    return pl is not None and isinstance(data, pl.DataFrame)


def _is_arrow_table(data) -> bool:
    try:
        import pyarrow as pa
        return isinstance(data, pa.Table)
    except Exception:  # pragma: no cover
        return False


def is_frame(data) -> bool:
    return isinstance(data, pd.DataFrame) or _is_polars_frame(data) or _is_arrow_table(data)


def do_dataframe_column_concatenation(data, column: List[str]):
    """Items of `column` naming a column contribute that column (cast to string, nulls
    -> ""); any other item is a literal separator (reference: sutro/common.py:72-108)."""
    try:
        if isinstance(data, pd.DataFrame):
            parts = []
            for p in column:
                if p in data.columns:
                    s = data[p].astype("string").fillna("")
                else:
                    s = pd.Series([p] * len(data), index=data.index, dtype="string")
                parts.append(s)
            out = parts[0]
            for s in parts[1:]:
                out = out.str.cat(s, na_rep="")
            return out.tolist()
        if _is_polars_frame(data):
            exprs = [pl.col(p).cast(pl.Utf8).fill_null("") if p in data.columns else pl.lit(p)
                     for p in column]
            return data.select(pl.concat_str(exprs, separator="", ignore_nulls=True)
                               .alias("concat"))["concat"].to_list()
        if _is_arrow_table(data):
            return do_dataframe_column_concatenation(data.to_pandas(), column)
        return None
    except Exception as e:
        raise ValueError(f"Error handling column concatentation: {e}")


def handle_data_helper(data, column: Union[str, List[str], None] = None):
    """list passthrough | frame column | multi-column concat | csv/parquet/txt path
    (reference: sutro/common.py:111-149).  `dataset-…` ids name server-side datasets and
    have no local meaning."""
    if isinstance(data, list):
        return data
    if is_frame(data):
        if column is None:
            raise ValueError("Column name must be specified for DataFrame input")
        if isinstance(column, list):
            return do_dataframe_column_concatenation(data, column)
        if _is_arrow_table(data):
            return data.column(column).to_pylist()
        return data[column].to_list() if hasattr(data[column], "to_list") else list(data[column])
    if isinstance(data, str):
        if data.startswith("dataset-"):
            raise ValueError("Sutro datasets live on the hosted service; the local engine takes "
                             "lists, DataFrames or csv/parquet/txt paths")
        ext = os.path.splitext(data)[1].lower()
        if ext in (".csv", ".parquet"):
            if column is None:
                raise ValueError("Column name must be specified for CSV/Parquet input")
            df = pd.read_csv(data) if ext == ".csv" else pd.read_parquet(data)
            return df[column].to_list()
        if ext in (".txt", ""):
            with open(data, "r") as f:
                return [line.strip() for line in f]
        raise ValueError(f"Unsupported file type: {ext}")
    raise ValueError("Unsupported data type. Please provide a list, DataFrame, or file path.")


def column_as_arrow(data, column: Union[str, List[str], None] = None):
    """The same inputs as `handle_data_helper`, but as ONE Arrow string column (pyarrow Array /
    ChunkedArray) whenever that can be had without creating a Python object per row: parquet
    and csv files are read by pyarrow straight into Arrow buffers, DataFrame / Table columns
    are converted by pyarrow's C++ loops.  The engine consumes the Arrow buffers directly
    (bytes + offsets go to the GPU as they are; engine.rows_to_blob), which is what matters at
    10^6 rows (BASELINE.json configs[3]).  Returns None when only the list path applies
    (lists, multi-column concatenation, .txt files): callers then use handle_data_helper.
    Argument errors are the reference's (sutro/common.py:117-147)."""
    try:
        import pyarrow as pa
    except Exception:  # pragma: no cover
        return None
    if isinstance(data, list) or isinstance(column, list):
        return None
    arr = None
    if isinstance(data, str) and not data.startswith("dataset-"):
        ext = os.path.splitext(data)[1].lower()
        if ext not in (".csv", ".parquet"):
            return None
        if column is None:
            raise ValueError("Column name must be specified for CSV/Parquet input")
        if ext == ".parquet":
            import pyarrow.parquet as pq
            arr = pq.read_table(data, columns=[column]).column(column)
        else:
            import pyarrow.csv as pacsv
            arr = pacsv.read_csv(data, convert_options=pacsv.ConvertOptions(
                include_columns=[column])).column(column)
    elif _is_arrow_table(data):
        if column is None:
            raise ValueError("Column name must be specified for DataFrame input")
        arr = data.column(column)
    elif isinstance(data, pd.DataFrame):
        if column is None:
            raise ValueError("Column name must be specified for DataFrame input")
        try:
            arr = pa.Array.from_pandas(data[column])
        except Exception:
            return None
    elif _is_polars_frame(data):
        if column is None:
            raise ValueError("Column name must be specified for DataFrame input")
        try:
            arr = data[column].to_arrow()
        except Exception:
            return None
    if arr is None:
        return None
    if not (pa.types.is_string(arr.type) or pa.types.is_large_string(arr.type)):
        try:
            arr = arr.cast(pa.large_string())        # numbers etc.: their text form
        except Exception:
            return None
    return arr


def normalize_output_schema(output_schema: Union[Dict[str, Any], Type[Any], None]):
    """BaseModel subclass -> .model_json_schema(); dict passthrough; else ValueError
    (reference: sutro/common.py:152-163)."""
    if hasattr(output_schema, "model_json_schema"):
        return output_schema.model_json_schema()
    if isinstance(output_schema, dict):
        return output_schema
    raise ValueError("Invalid output schema type. Must be a dictionary or a pydantic Model.")


def check_penalties(presence_penalty=0.0, frequency_penalty=0.0, repetition_penalty=1.0,
                    min_p=0.0) -> Tuple[float, float, float, float]:
    """vLLM's ranges for its sampling parameters of the same names (ValueError outside them);
    returns them as floats.  Neutral: presence 0, frequency 0, repetition 1, min_p 0."""
    p, f, r, m = (float(x) for x in (presence_penalty, frequency_penalty, repetition_penalty,
                                     min_p))
    if not -2.0 <= p <= 2.0:
        raise ValueError(f"presence_penalty must be in [-2, 2], got {p}")
    if not -2.0 <= f <= 2.0:
        raise ValueError(f"frequency_penalty must be in [-2, 2], got {f}")
    if not (r > 0.0 and math.isfinite(r)):
        raise ValueError(f"repetition_penalty must be > 0, got {r}")
    if not 0.0 <= m <= 1.0:
        raise ValueError(f"min_p must be in [0, 1], got {m}")
    return p, f, r, m
