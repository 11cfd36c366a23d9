"""`Sutro` — the local, H100-native counterpart of the reference SDK client for the
infer() hot path (reference: sutro/sdk.py:46, `class Sutro`).

Drop-in surface (same names, positional order, defaults, return and error
conventions as the reference):
  infer()                 sutro/sdk.py:434-502   -> job-id str | None
  infer_per_model()       sutro/sdk.py:655-757   -> list[str]
  await_job_completion()  sutro/sdk.py:1493-1568 -> DataFrame | None
  get_job_results()       sutro/sdk.py:1037-1190 -> DataFrame (JSON top-level unpack)
  get_job_status() / fetch_job() / list_jobs() / cancel_job()
What changes is what happens at the reference's single process boundary
(`do_request("POST", "batch-inference")`, sutro/sdk.py:223): instead of shipping the
column to a hosted service, the rows go through `engine.LocalEngine.generate` on this
machine's H100(s).  Jobs complete before infer() returns, so the polling helpers
resolve immediately; results are kept in memory and (like the reference,
sutro/sdk.py:1065-1117) cached as snappy parquet under ~/.sutro/job-results/.

Conventions kept from the reference: bad arguments raise ValueError; engine/service
failures print a message and return None; pandas input is updated in place with
`output_column`, other frames are left untouched; outputs are positional.
"""
from __future__ import annotations

import json
import os
import time
import uuid
from typing import Any, Dict, List, Optional, Type, Union

import numpy as np
import pandas as pd

from .common import (ModelOptions, check_penalties, column_as_arrow, handle_data_helper,
                     is_frame,
                     normalize_output_schema, pl, to_colored_text)
from .interfaces import BaseSutroClient, JobStatus
from .templates import Templates

JOB_NAME_CHAR_LIMIT = 45          # sutro/sdk.py:39-40
JOB_DESCRIPTION_CHAR_LIMIT = 512


class _Job:
    def __init__(self, job_id, model, n_rows, name, description, priority):
        self.job_id, self.model, self.n_rows = job_id, model, n_rows
        self.name, self.description, self.priority = name, description, priority
        self.status = JobStatus.QUEUED
        self.inputs: Optional[List[str]] = None
        self.outputs: Optional[list] = None
        self.embeddings = None
        self.stats: Dict[str, Any] = {}
        self.failure_reason: Optional[str] = None
        self.cum_logprobs = None
        self.confidence = None
        self.progress: Dict[str, Any] = {}
        self.created = time.time()
        self.cost_estimate: Optional[float] = None


class _ProgressStream:
    """Turns the engine's (rows_done, input_tokens, output_tokens) callback into the records
    the reference reads from `stream-job-progress/{id}` (sutro/sdk.py:331-358):
    `{"update_type": "progress", "result": rows_done}` and `{"update_type": "tokens",
    "result": {input_tokens, output_tokens, total_tokens_processed_per_second}}`.  Records
    go to `sink` (the client's `on_progress` hook) and, when `bar` is set, drive a tqdm bar
    with the reference's postfix text; counters are merged monotonically like the reference
    does."""

    def __init__(self, job: _Job, sink=None, bar: bool = False):
        self.job, self.sink = job, sink
        self.t0 = time.perf_counter()
        self.state = {"input_tokens": 0, "output_tokens": 0, "total_tokens_processed_per_second": 0}
        self.rows = 0
        self.pbar = None
        if bar:
            try:
                from tqdm import tqdm
                self.pbar = tqdm(total=job.n_rows, desc="Progress",
                                 postfix="Input tokens processed: 0")
            except Exception:
                self.pbar = None

    def __call__(self, rows_done: int, input_tokens: int, output_tokens: int) -> None:
        dt = max(time.perf_counter() - self.t0, 1e-9)
        records = [{"update_type": "progress", "result": int(rows_done)},
                   {"update_type": "tokens",
                    "result": {"input_tokens": int(input_tokens),
                               "output_tokens": int(output_tokens),
                               "total_tokens_processed_per_second":
                                   round((input_tokens + output_tokens) / dt, 1)}}]
        self.rows = max(self.rows, int(rows_done))
        for k, v in records[1]["result"].items():
            if k == "total_tokens_processed_per_second" or v >= self.state[k]:
                self.state[k] = v
        self.job.progress = {"rows_done": self.rows, **self.state}
        if self.sink is not None:
            for r in records:
                self.sink(r)
        if self.pbar is not None:
            if self.rows > self.pbar.n:
                self.pbar.update(self.rows - self.pbar.n)
            self.pbar.postfix = (f"Input tokens processed: {self.state['input_tokens']}, Output "
                                 f"tokens generated: {self.state['output_tokens']}, Total tokens/s: "
                                 f"{self.state['total_tokens_processed_per_second']}")
            self.pbar.refresh()

    def close(self):
        if self.pbar is not None:
            self.pbar.close()
            self.pbar = None


class Sutro(Templates, BaseSutroClient):
    def __init__(self, devices: Optional[List[int]] = None, weights_seed: int = 0,
                 engine_options: Optional[Dict[str, Any]] = None, cache_dir: Optional[str] = None,
                 verbose: bool = True, on_progress=None,
                 model_paths: Optional[Dict[str, str]] = None, fsm_limits=None):
        self.devices = devices or [0]
        # schema_fsm.FsmLimits: bounds for what a JSON schema leaves open (strings without
        # maxLength stop at 64 characters, arrays without maxItems at 8 items, ... by default —
        # the hosted service has no such caps; raise them here when outputs need the room)
        self.fsm_limits = fsm_limits
        # model name -> Hugging Face model directory (config.json, tokenizer.json, *.safetensors);
        # models without a path run on seeded random weights and the synthetic vocabulary
        self.model_paths = dict(model_paths or {})
        # optional callable(record): receives every progress / tokens record of a running job
        self.on_progress = on_progress
        self.weights_seed = weights_seed
        self.engine_options = dict(engine_options or {})
        self.cache_dir = os.path.expanduser(cache_dir or "~/.sutro/job-results")
        self.verbose = verbose
        self._engines: Dict[str, Any] = {}
        self._jobs: Dict[str, _Job] = {}

    # ------------------------------------------------------------------ engines
    def _say(self, msg: str, state: str = None):
        if self.verbose:
            print(to_colored_text(msg, state))

    def _engine(self, model: str):
        base = model[:-len("-thinking")] if str(model).endswith("-thinking") else model
        if model not in self._engines and model not in self.model_paths and (
                base in self._engines or base in self.model_paths):
            model = base          # "<model>-thinking" is the same weights, another turn format
        if model not in self._engines and model in self.model_paths:
            from .pretrained import load_pretrained
            if len(self.devices) > 1:
                raise ValueError("model_paths with several devices is not supported yet: "
                                 "run one process per GPU")
            self._say(f"Loading {model} from {self.model_paths[model]} on cuda:{self.devices[0]}")
            self._engines[model] = load_pretrained(self.model_paths[model], self.devices[0],
                                                   name=model, **self.engine_options)
        if model not in self._engines:
            model = base
        if model not in self._engines:
            from .engine import LocalEngine, MultiGpuEngine
            where = ", ".join(f"cuda:{d}" for d in self.devices)
            self._say(f"Loading {model} on {where} (random-init weights, seed "
                      f"{self.weights_seed}: no checkpoints are available offline)")
            if len(self.devices) > 1:   # one replica per GPU, rows sharded across them
                self._engines[model] = MultiGpuEngine.from_seed(
                    model, self.devices, seed=self.weights_seed, **self.engine_options)
            else:
                self._engines[model] = LocalEngine.from_seed(model, seed=self.weights_seed,
                                                             device=self.devices[0],
                                                             **self.engine_options)
        return self._engines[model]

    @staticmethod
    def _default_max_new_tokens(eng, json_schema, thinking_chars=None, limits=None) -> int:
        """Output budget when sampling_params names none.  Schema jobs: the longest string the
        schema's automaton accepts (every token is at least one byte), so a constrained row
        can always close its object — a row cut mid-object would not be JSON.  Free text: 512."""
        spec = getattr(eng, "spec", None)
        # half the window, but no more than 2,048 tokens: a job's default budget does not grow
        # with the context window
        cap = max(16, min(getattr(spec, "max_position", 4096), 4096) // 2)
        if thinking_chars is not None and hasattr(eng, "compile_schema"):
            longest = eng.compile_schema(json_schema, limits, int(thinking_chars)).longest_path()
            return int(min(max(longest, 8), cap)) if longest is not None else \
                int(min(512 + 4 * int(thinking_chars), cap))
        if json_schema is not None and hasattr(eng, "compile_schema"):
            longest = eng.compile_schema(json_schema, limits).longest_path()
            if longest is not None:
                return int(min(max(longest, 8), cap))
        return int(min(512, cap))

    def _dispatch(self, eng, input_data, kw):
        """The reference's one process boundary (`POST batch-inference`, sutro/sdk.py:223) as a
        local call.  One GPU: `sb200_infer_text`, one C call with host buffers.  One process per
        GPU under torchrun: the row-sharded path (sharding.infer_frame_sharded; rank 0 holds the
        frame and receives the ordered results).  Several devices in this process:
        MultiGpuEngine."""
        import types
        try:
            import torch.distributed as dist
            sharded = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        except Exception:
            sharded = False
        if sharded and hasattr(eng, "run_blob_dev"):
            from .sharding import infer_frame_sharded
            kw = dict(kw)
            progress = kw.pop("progress", None)
            out = infer_frame_sharded(eng, input_data if dist.get_rank() == 0 else None, src=0,
                                      progress=progress, **kw)
            if out is None:
                return None
            return types.SimpleNamespace(outputs=out.get("outputs"), embeddings=out.get("embeddings"),
                                         stats=out["stats"], cum_logprobs=None)
        if hasattr(eng, "infer_one_call"):
            return eng.infer_one_call(input_data, return_tokens=False, **kw)
        if not isinstance(input_data, list):      # engines without the Arrow-aware entry points
            input_data = input_data.to_pylist()
        return eng.generate(input_data, **kw)

    def register_engine(self, model: str, engine) -> None:
        """Use a pre-built LocalEngine (tests, benchmarks, multi-GPU workers)."""
        self._engines[model] = engine

    # ------------------------------------------------------------------ the hot path
    def _run_one_batch_inference(self, data, model, column, output_column, job_priority,
                                 json_schema, sampling_params, system_prompt, cost_estimate,
                                 stay_attached, random_seed_per_input, truncate_rows, name,
                                 description):
        if name is not None and len(name) > JOB_NAME_CHAR_LIMIT:
            raise ValueError(f"Job name cannot exceed {JOB_NAME_CHAR_LIMIT} characters.")
        if description is not None and len(description) > JOB_DESCRIPTION_CHAR_LIMIT:
            raise ValueError(
                f"Job description cannot exceed {JOB_DESCRIPTION_CHAR_LIMIT} characters.")
        # files and frame columns travel as Arrow buffers (no Python object per row); lists,
        # multi-column concatenations and .txt files take the reference's list path
        input_data = column_as_arrow(data, column)
        if input_data is None:
            input_data = handle_data_helper(data, column)
        # sampling_params is an opaque dict in the reference (forwarded as is, sdk.py:203);
        # the local engine understands the usual keys and rejects the rest loudly.
        sp = dict(sampling_params or {})
        known = {"temperature", "top_p", "top_k", "seed", "random_seed", "max_tokens",
                 "max_new_tokens", "ignore_eos", "max_thinking_chars", "presence_penalty",
                 "frequency_penalty", "repetition_penalty", "min_p"}
        unknown = sorted(set(sp) - known)
        if unknown:
            raise ValueError(f"unsupported sampling_params for the local engine: {unknown} "
                             f"(supported: {sorted(known)})")
        temperature = float(sp.get("temperature") or 0.0)
        top_p = float(sp.get("top_p") if sp.get("top_p") is not None else 1.0)
        top_k = int(sp.get("top_k") if sp.get("top_k") not in (None, -1) else 0)
        if temperature < 0 or not (0.0 < top_p <= 1.0) or top_k < 0:
            raise ValueError("sampling_params: temperature >= 0, 0 < top_p <= 1, top_k >= 0")
        seed = int(sp.get("seed", sp.get("random_seed", 0)) or 0)
        # vLLM's keys and ranges (None = the neutral value, as vLLM reads it)
        penalties = dict(zip(
            ("presence_penalty", "frequency_penalty", "repetition_penalty", "min_p"),
            check_penalties(*(sp[k] if sp.get(k) is not None else d for k, d in (
                ("presence_penalty", 0.0), ("frequency_penalty", 0.0),
                ("repetition_penalty", 1.0), ("min_p", 0.0))))))
        max_new = sp.get("max_tokens", sp.get("max_new_tokens"))
        max_new = None if max_new is None else int(max_new)

        job = _Job("job-" + uuid.uuid4().hex[:24], model, len(input_data), name, description,
                   job_priority)
        self._jobs[job.job_id] = job
        name_text = f" and name {name}" if name is not None else ""
        self._say(f"🛠 Priority {job_priority} Job created with ID: {job.job_id}{name_text}",
                  "success")
        self._say(f"Model: {model}")
        try:
            eng = self._engine(model)
            job.status = JobStatus.RUNNING
            if cost_estimate:
                # dry run: count input tokens only (the reference asks the service for a
                # dollar estimate; locally the marginal cost is zero)
                as_list = input_data if isinstance(input_data, list) else input_data.to_pylist()
                toks = eng.tokenizer.encode([("" if x is None else str(x)) for x in as_list])
                job.stats = {"input_tokens": sum(map(len, toks))}
                job.cost_estimate = 0.0
                job.status = JobStatus.SUCCEEDED
                self._say(f"✔ Cost estimates retrieved for job {job.job_id}: $0.0 "
                          f"({job.stats['input_tokens']} input tokens)", "success")
                return job.job_id
            # "<model>-thinking" (sutro/common.py:28-32): reason first, answer after </think>; the
            # job's outputs are {"content", "reasoning_content"} objects (sutro/sdk.py:1155-1164)
            thinking = None
            if str(model).endswith("-thinking") and not getattr(eng.spec, "embedding_model", False):
                thinking = int(sp.get("max_thinking_chars", 128))
            if max_new is None:
                max_new = self._default_max_new_tokens(eng, json_schema, thinking, self.fsm_limits)
            t0 = time.perf_counter()
            stream = None
            if self.on_progress is not None or (stay_attached and self.verbose):
                stream = _ProgressStream(job, self.on_progress,
                                         bar=bool(stay_attached and self.verbose))
            kw = dict(system_prompt=system_prompt, json_schema=json_schema,
                      max_new_tokens=max_new, ignore_eos=bool(sp.get("ignore_eos", False)),
                      truncate_rows=truncate_rows, temperature=temperature, top_k=top_k,
                      top_p=top_p, seed=seed, seed_per_row=bool(random_seed_per_input),
                      return_logprobs=True, progress=stream)
            # only non-neutral values are passed: engines without them keep working
            kw.update({k: v for k, v in penalties.items()
                       if v != (1.0 if k == "repetition_penalty" else 0.0)})
            if thinking is not None:
                kw["thinking_chars"] = thinking
            if self.fsm_limits is not None:
                kw["fsm_limits"] = self.fsm_limits
            res = self._dispatch(eng, input_data, kw)
            if res is None:          # a non-source rank of a row-sharded job: nothing to report
                job.status = JobStatus.SUCCEEDED
                job.outputs = []
                return job.job_id
            dt = time.perf_counter() - t0
            if stream is not None:
                stream.close()
        except KeyboardInterrupt:
            job.status = JobStatus.CANCELLED
            return None
        except ValueError:
            job.status = JobStatus.FAILED
            raise
        except Exception as e:  # engine failure: print + None, like a non-200 (sdk.py:225-234)
            job.status, job.failure_reason = JobStatus.FAILED, str(e)
            self._say(f"Error: {e}", "fail")
            return None
        job.inputs = input_data
        job.stats = res.stats
        job.cum_logprobs = getattr(res, "cum_logprobs", None)
        if json_schema is not None and job.cum_logprobs is not None:
            # Schema-constrained job: the sampler's log-probabilities are taken over the
            # schema-valid tokens only (forced tokens contribute 0), so exp(sum) is the
            # probability of this output among all outputs the schema admits — for an enum
            # field, the model's probability of the chosen label.
            job.confidence = np.exp(np.asarray(job.cum_logprobs, dtype=np.float64))
        if res.embeddings is not None:
            # one fp32 [n_rows, d] array; the per-row "outputs" are views into it (a million
            # rows must not become a billion Python floats)
            job.embeddings = res.embeddings
            job.outputs = list(res.embeddings)
        else:
            job.outputs = res.outputs
            if thinking is not None and job.outputs is not None:
                from .schema_fsm import split_thinking
                shaped = []
                for text in job.outputs:
                    reasoning, content = split_thinking(text)
                    if json_schema is not None:
                        try:
                            content = json.loads(content)
                        except ValueError:
                            pass       # cut by max_tokens: keep the text
                    shaped.append(json.dumps({"content": content, "reasoning_content": reasoning},
                                             ensure_ascii=False))
                job.outputs = shaped
        job.status = JobStatus.SUCCEEDED
        tps = (res.stats.get("input_tokens", 0) + res.stats.get("output_tokens", 0)) / max(dt, 1e-9)
        self._say(f"Input tokens processed: {res.stats.get('input_tokens', 0)}, Output tokens "
                  f"generated: {res.stats.get('output_tokens', 0)}, Total tokens/s: {tps:.0f}")
        if not stay_attached:
            self._say(f"Use `so.get_job_status('{job.job_id}')` to check the status of the job")
            return job.job_id
        # attached: preview + positional write-back (sdk.py:406-430)
        results = job.outputs
        if is_frame(data):
            if isinstance(data, pd.DataFrame):
                data[output_column] = results
                preview = data
            elif pl is not None and isinstance(data, pl.DataFrame):
                preview = data.with_columns(pl.Series(output_column, results))
            else:
                preview = data.append_column(output_column, [results])
            if self.verbose:
                print(preview)
            self._say("✔ Displaying result preview. You can join the results on the original "
                      f"dataframe with `so.get_job_results('{job.job_id}', "
                      "with_original_df=<original_df>)`", "success")
        else:
            if self.verbose:
                print(results if len(results) <= 20 else results[:20] + ["..."])
            self._say("✔ Job results received. You can re-obtain the results with "
                      f"`so.get_job_results('{job.job_id}')`", "success")
        return job.job_id

    def infer(
        self,
        data,
        model: ModelOptions = "gemma-3-12b-it",
        name: Optional[str] = None,
        description: Optional[str] = None,
        column: Union[str, List[str]] = None,
        output_column: str = "inference_result",
        job_priority: int = 0,
        output_schema: Union[Dict[str, Any], Type[Any]] = None,
        sampling_params: dict = None,
        system_prompt: str = None,
        dry_run: bool = False,
        stay_attached: Optional[bool] = None,
        random_seed_per_input: bool = False,
        truncate_rows: bool = True,
    ):
        """Run inference over `data` on the local H100 engine; returns the job id."""
        model = self._resolve_model(model)
        if stay_attached is None:
            stay_attached = job_priority == 0
        json_schema = None
        if output_schema:
            json_schema = normalize_output_schema(output_schema)
        return self._run_one_batch_inference(data, model, column, output_column, job_priority,
                                             json_schema, sampling_params, system_prompt, dry_run,
                                             stay_attached, random_seed_per_input, truncate_rows,
                                             name, description)

    # the reference's default model is served by its hosted service only; scripts that rely on
    # the default keep working here on the local flagship
    LOCAL_DEFAULT_MODEL = "qwen-3-4b"

    def _resolve_model(self, model: str) -> str:
        from . import modelspec as MS
        if model in self._engines or model in self.model_paths:
            return model
        try:
            MS.get_spec(model)
            return model
        except ValueError:
            if model == "gemma-3-12b-it":
                self._say(f"Model {model!r} (the hosted service's default) has no local engine; "
                          f"running {self.LOCAL_DEFAULT_MODEL!r} instead")
                return self.LOCAL_DEFAULT_MODEL
            raise ValueError(f"Unknown model {model!r}: local engines exist for "
                             f"{sorted(MS.SPECS)} and for directories named in model_paths "
                             f"({sorted(self.model_paths)})")

    def infer_per_model(self, data, models: List[ModelOptions], names: List[str] = None,
                        descriptions: List[str] = None, column=None,
                        output_column: str = "inference_result", job_priority: int = 0,
                        output_schema=None, sampling_params: dict = None, system_prompt: str = None,
                        dry_run: bool = False, random_seed_per_input: bool = False,
                        truncate_rows: bool = True) -> List[str]:
        """One detached job per model (reference: sutro/sdk.py:655-757)."""
        names = names if isinstance(names, list) else [None] * len(models)
        descriptions = descriptions if isinstance(descriptions, list) else [None] * len(models)
        if len(names) != len(models) or len(descriptions) != len(models):
            raise ValueError("names/descriptions must match the number of models")
        return [self.infer(data, m, names[i], descriptions[i], column, output_column, job_priority,
                           output_schema, sampling_params, system_prompt, dry_run, False,
                           random_seed_per_input, truncate_rows) for i, m in enumerate(models)]

    # ------------------------------------------------------------------ job surface
    def _job(self, job_id: str) -> _Job:
        if job_id not in self._jobs:
            raise ValueError(f"Unknown job id {job_id}")
        return self._jobs[job_id]

    def get_job_status(self, job_id: str) -> JobStatus:
        return self._job(job_id).status

    def fetch_job(self, job_id: str) -> Dict[str, Any]:
        j = self._job(job_id)
        return {"job_id": j.job_id, "status": j.status.value, "model": j.model, "name": j.name,
                "description": j.description, "num_rows": j.n_rows, "job_priority": j.priority,
                "input_tokens": j.stats.get("input_tokens"),
                "output_tokens": j.stats.get("output_tokens"), "failure_reason": j.failure_reason,
                "cost_estimate": j.cost_estimate, "datetime_created": j.created}

    def list_jobs(self) -> List[Dict[str, Any]]:
        return [self.fetch_job(j) for j in self._jobs]

    def cancel_job(self, job_id: str):
        j = self._job(job_id)
        if not j.status.is_terminal():
            j.status = JobStatus.CANCELLED
        return {"job_id": job_id, "status": j.status.value}

    def await_job_completion(self, job_id: str, timeout: Optional[int] = 7200,
                             obtain_results: bool = True, output_column: str = "inference_result",
                             is_cost_estimate: bool = False):
        """Local jobs are already terminal when infer() returns; this resolves the job id
        to its results frame exactly like the reference (sutro/sdk.py:1493-1568)."""
        status = self.get_job_status(job_id)
        if status == JobStatus.SUCCEEDED:
            self._say("Job completed! Retrieving results..." if obtain_results
                      else "Job completed!", "success")
            if obtain_results and not is_cost_estimate:
                return self.get_job_results(job_id, output_column=output_column)
            return None
        if status == JobStatus.FAILED:
            self._say("Job has failed", "fail")
        elif status == JobStatus.CANCELLED:
            self._say("Job has been cancelled")
        return None

    def get_job_results(self, job_id: str, include_inputs: bool = False,
                        include_cumulative_logprobs: bool = False, with_original_df=None,
                        output_column: str = "inference_result", disable_cache: bool = False,
                        unpack_json: bool = True):
        """Results frame with the reference's column contract (sutro/sdk.py:1037-1190):
        [inputs] / <output_column>, JSON outputs fanned out to top-level keys when the
        first row parses as a JSON object.  Returns a pandas DataFrame (polars when the
        original frame is polars and polars is installed)."""
        j = self._job(job_id)
        if j.status != JobStatus.SUCCEEDED or j.outputs is None:
            self._say(f"Job {job_id} has no results (status {j.status.value})", "fail")
            return None
        if include_cumulative_logprobs and j.cum_logprobs is None:
            raise ValueError("this job recorded no cumulative logprobs (embedding job?)")
        path = os.path.join(self.cache_dir, f"{job_id}.snappy.parquet")
        cols: Dict[str, Any] = {}
        if include_inputs:
            cols["inputs"] = j.inputs if isinstance(j.inputs, list) else j.inputs.to_pylist()
        cols[output_column] = j.outputs
        if include_cumulative_logprobs:
            cols["cumulative_logprobs"] = [float(x) for x in j.cum_logprobs]
        if j.confidence is not None:   # kept whenever the job produced one (sdk.py:1122-1127)
            cols["confidence_score"] = [float(x) for x in j.confidence]
        df = pd.DataFrame(cols)
        if not disable_cache:
            try:
                os.makedirs(self.cache_dir, exist_ok=True)
                if j.embeddings is not None:
                    import pyarrow as pa
                    import pyarrow.parquet as pq
                    emb = j.embeddings
                    vec = pa.FixedSizeListArray.from_arrays(pa.array(emb.reshape(-1)), emb.shape[1])
                    names, arrays = [output_column], [vec]
                    if include_inputs:
                        names, arrays = ["inputs"] + names, [pa.array(cols["inputs"])] + arrays
                    pq.write_table(pa.table(arrays, names=names), path, compression="snappy")
                else:
                    df.to_parquet(path, compression="snappy")
            except Exception as e:  # cache is best effort
                self._say(f"(results cache not written: {e})")
        if unpack_json and len(df) and isinstance(df[output_column].iloc[0], str):
            try:
                first = json.loads(df[output_column].iloc[0])
                if isinstance(first, dict):
                    def _loads(x):   # a row that is not JSON (cut by max_tokens) unpacks to None
                        try:
                            return json.loads(x)
                        except (TypeError, ValueError):
                            return None
                    decoded = [_loads(x) for x in df[output_column]]
                    for key in first.keys():
                        df[key] = [d.get(key) if isinstance(d, dict) else None for d in decoded]
                    if sorted(first.keys()) == ["content", "reasoning_content"] and \
                            isinstance(first["content"], dict):
                        for key in first["content"].keys():
                            df[key] = [d["content"].get(key)
                                       if isinstance(d, dict) and isinstance(d.get("content"), dict)
                                       else None for d in decoded]
                        df = df.drop(columns=["content"])
                    if output_column not in first:   # a key may reuse the column's name (rank)
                        df = df.drop(columns=[output_column])
            except Exception:
                pass  # first row is not JSON: leave the column as text (sdk.py:1168-1170)
        if with_original_df is not None:
            if isinstance(with_original_df, pd.DataFrame):
                out = with_original_df.copy()
                for c in df.columns:
                    out[c] = df[c].values
                return out
            if pl is not None and isinstance(with_original_df, pl.DataFrame):
                return with_original_df.with_columns(pl.from_pandas(df))
        return df

    def get_job_embeddings(self, job_id: str):
        """fp32 [n_rows, d] array for embedding-model jobs (zero-copy alternative to the
        list-of-lists results column)."""
        return self._job(job_id).embeddings

    # quotas / datasets / auth are properties of the hosted service, not of this path; the
    # calls scripts written for the reference make at start-up are accepted and do nothing
    def try_authentication(self, api_key: str = None):
        return {"authenticated": True, "backend": "local-b200"}

    def set_api_key(self, api_key: str):                 # sutro/sdk.py:58-71
        self.api_key = api_key

    def set_base_url(self, base_url: str):               # sutro/sdk.py:73-83
        self.base_url = base_url

    def set_serving_base_url(self, serving_base_url: str):
        self.serving_base_url = serving_base_url

    def get_quotas(self):                                # sutro/sdk.py:1477-1491
        return [{"job_priority": p, "row_quota": None, "token_quota": None} for p in (0, 1)]

    def attach(self, job_id):                            # sutro/sdk.py:759-870
        """Jobs run synchronously here, so attaching reports the final state."""
        j = self._job(job_id)
        self._say(f"Job {job_id}: {j.status.value} ({j.n_rows} rows)",
                  "success" if j.status == JobStatus.SUCCEEDED else None)
        return j.status

    def _no_datasets(self, *a, **kw):
        raise NotImplementedError("datasets are a feature of the hosted service; pass lists, "
                                  "DataFrames or csv / parquet / txt paths to infer()")

    create_dataset = upload_to_dataset = list_datasets = list_dataset_files = \
        download_from_dataset = _no_datasets
