"""sutro_b200 — H100-native local backend for the sutro.infer() hot path.

    import sutro_b200 as so
    job_id = so.infer(df, column="review", model="qwen-3-4b",
                      system_prompt="...", output_schema=Sentiment)
    results = so.get_job_results(job_id, with_original_df=df)

Like the reference package (sutro/__init__.py:4-9) the module-level functions are the
bound methods of one process-wide `Sutro()` instance; it is created lazily so that
importing the package needs neither a GPU nor the compiled library.
"""
from __future__ import annotations

__version__ = "0.1.0"

from .interfaces import BaseSutroClient, JobStatus  # noqa: F401
from .sdk import Sutro  # noqa: F401

_instance = None
_PUBLIC = ["infer", "infer_per_model", "await_job_completion", "get_job_results",
           "get_job_status", "fetch_job", "list_jobs", "cancel_job", "get_job_embeddings",
           "register_engine", "classify", "embed", "score", "rank", "elo", "attach",
           "set_api_key", "set_base_url", "set_serving_base_url", "get_quotas",
           "try_authentication"]


def _client() -> Sutro:
    global _instance
    if _instance is None:
        _instance = Sutro()
    return _instance


def configure(**kwargs) -> Sutro:
    """(Re)create the process-wide client with constructor options — `devices`,
    `engine_options` (max_position, max_slots, max_prefill_tokens, kv_pages, ...), `model_paths`, `verbose`,
    `cache_dir`, `on_progress`, `fsm_limits` (see `Sutro.__init__`).  The reference configures its singleton
    through setters (set_api_key / set_base_url, sutro/sdk.py:58-95); a local engine's knobs
    are construction-time."""
    global _instance
    _instance = Sutro(**kwargs)
    return _instance


def _bind(name):
    def call(*a, **kw):
        return getattr(_client(), name)(*a, **kw)
    call.__name__ = name
    call.__doc__ = getattr(Sutro, name).__doc__
    return call


for _n in _PUBLIC:
    globals()[_n] = _bind(_n)

__all__ = _PUBLIC + ["Sutro", "JobStatus", "BaseSutroClient", "configure"]
