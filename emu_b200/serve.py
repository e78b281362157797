"""Serving shell: the reference demo's HTTP contract over a request-batching scheduler (SURVEY.md §8f-4).

Replaces Emu2/demo/backend/pytorch_model/backend.py.  The contract the demo's front end speaks is kept field for field:

    POST /v1/mmc   chat          form: log_id, prompt = JSON [[type, payload], ...] ("TEXT" -> the string itself, any other type
                                 -> the NAME of an uploaded file holding the picture), do_sample, max_new_tokens (10),
                                 temperature (0.7), top_k (3), top_p (0.9), length_penalty (1), num_beams (5),
                                 repetition_penalty (1.0)                                            backend.py:167-214
    POST /v1/mmg   generation    form: log_id, prompt (same encoding), classifier_free_guidance, steps  backend.py:112-134
    response       JSON {"code": 0, "data": <text | base64 WEBP>}  or  {"code": -1, "data": <error message>}
                                                                                              backend.py:131-150,203-226

What is different is what sits behind it.  The reference keeps a pool of `concurrency` pipelines behind a semaphore
(backend.py:55-93): one request per pipeline at a time, every request a batch-1 generate call — on the decode path that is one
full pass over the 65 GB of LLaMA weights per token PER REQUEST.  Here every pipeline has one scheduler thread that owns it (the
engine is single-host-thread by contract, include/emu_b200.h) and admits requests in batches: whatever is waiting with the same
decoding knobs when the pipeline becomes free is sent through ONE `forward_batch` call (left-padded prompts / stacked latents),
so concurrent requests share each weight pass.  Admission is per generate call, not per decode step: the engine advances all
cache rows in lock-step (one `cur_len`), so a request cannot join a batch that is already decoding — it waits for the next one.

Opt-in continuous batching for chat (`EmuServer(chat_scheduler="continuous")`, `--continuous-batching`): a ContinuousWorker
runs the pipeline's model under emu_b200/batching.py's SlotScheduler instead — requests join the decode batch between two
steps and leave it as soon as they are finished, each with its own knobs.  Single GPU only.  The same for image generation
(`EmuServer(generate_scheduler="continuous")`, `--continuous-generation`): a ContinuousWorker drives a DenoiseSlotScheduler,
whose latent slots join and leave between UNet steps, each request with its own step count and guidance.  With
`generate_encode_steps=R` (`--generate-encode-steps R`) the newcomers' prompts are encoded together in LLaMA regression slots,
at most R regression steps between two UNet steps, instead of one whole generate_image per newcomer while the live slots wait.

With tensor parallelism (launched under torchrun, one process per GPU) rank 0 serves HTTP and broadcasts every admitted batch;
the other ranks run `follow()` and execute the same calls, which is what the engine's collectives need.

Python standard library only (http.server + email for multipart parsing): Flask, which the reference uses, is not a dependency.
"""
import argparse
import base64
import io
import json
import logging
import os
import os.path as osp
import queue
import threading
import time
import traceback
from email.parser import BytesParser
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from urllib.parse import parse_qs

log = logging.getLogger("emu_b200.serve")

CHAT_DEFAULTS = dict(do_sample=False, max_new_tokens=10, temperature=0.7, top_k=3, top_p=0.9, length_penalty=1.0,
                     num_beams=5, repetition_penalty=1.0)                       # backend.py:187-194


class _Request:
    __slots__ = ("inputs", "knobs", "log_id", "done", "result", "error", "t_in")

    def __init__(self, inputs, knobs, log_id=""):
        self.inputs, self.knobs, self.log_id = inputs, knobs, log_id
        self.done = threading.Event()
        self.result = self.error = None
        self.t_in = time.time()

    def key(self):
        return tuple(sorted(self.knobs.items()))


class BatchingWorker(threading.Thread):
    """One pipeline, one thread that owns it, one queue in front.

    `pipeline` is an EmuChatGeneration / EmuVisualGeneration (anything with the reference's call signature; `forward_batch`
    is used when present, otherwise the requests of a batch run one after the other).  `max_batch(knobs) -> int` bounds a batch
    (chat: KV-cache rows // num_beams; generation: latents per denoise loop).  `max_wait_ms`: how long the first request of a
    batch waits for company when the queue is otherwise empty — 0 = never wait, only batch what is already there.
    `announce(kind, batch_inputs, knobs)` is called before every batch (tensor parallel: broadcast to the follower ranks)."""

    def __init__(self, pipeline, kind, max_batch=None, max_wait_ms=0.0, announce=None, name=None):
        super().__init__(daemon=True, name=name or ("emu-%s-worker" % kind))
        self.pipeline, self.kind = pipeline, kind
        self.max_batch = max_batch or (lambda knobs: 1)
        self.max_wait = max_wait_ms / 1000.0
        self.announce = announce
        self.q = queue.Queue()
        self.held = []                       # admitted to nothing yet: requests whose knobs did not match the current batch
        self.batches = []                    # sizes of the batches run so far (observability; the tests read it)
        self._halt = threading.Event()

    # ---- producer side (HTTP handler threads) ----
    def load(self):
        """requests waiting in front of this worker (EmuServer sends a request to the least loaded one)"""
        return self.q.qsize() + len(self.held)

    def submit(self, inputs, knobs, log_id="", timeout=None):
        r = _Request(inputs, knobs, log_id)
        self.q.put(r)
        if not r.done.wait(timeout):
            raise TimeoutError("request %s timed out in the queue" % log_id)
        if r.error is not None:
            raise r.error
        return r.result

    def stop(self):
        self._halt.set()
        self.q.put(None)

    # ---- consumer side ----
    def _next_batch(self):
        """first waiting request + everything compatible with it that is already queued (or arrives within max_wait),
        oldest first; incompatible requests keep their place in line for the next batch"""
        first = self.held.pop(0) if self.held else self.q.get()
        if first is None:
            return None
        batch, key, cap = [first], first.key(), max(1, int(self.max_batch(first.knobs)))
        keep = []
        for r in self.held:
            (batch if (r.key() == key and len(batch) < cap) else keep).append(r)
        self.held = keep
        deadline = time.time() + self.max_wait
        while len(batch) < cap:
            try:
                wait = deadline - time.time()
                r = self.q.get(timeout=wait) if wait > 0 else self.q.get_nowait()
            except queue.Empty:
                break
            if r is None:
                self._halt.set()
                break
            (batch if r.key() == key else self.held).append(r)
        return batch

    def _run_batch(self, batch):
        knobs = batch[0].knobs
        inputs = [r.inputs for r in batch]
        if self.announce is not None:
            self.announce(self.kind, inputs, knobs)
        if len(batch) > 1 and hasattr(self.pipeline, "forward_batch"):
            outs = list(self.pipeline.forward_batch(inputs, **knobs))
        else:
            outs = [self.pipeline(inputs=i, **knobs) for i in inputs]
        if len(outs) != len(batch):
            raise RuntimeError("pipeline returned %d results for %d requests" % (len(outs), len(batch)))
        return outs

    def _settle(self, batch):
        """run the batch; a request fails on its own account only: when a shared call raises, its requests are retried one
        by one, so that one bad prompt does not answer `code -1` to the callers it happened to be batched with"""
        try:
            for r, o in zip(batch, self._run_batch(batch)):
                r.result = o
        except Exception as ex:  # the request fails, the server lives (backend.py:141-146)
            log.error("%s batch of %d failed: %s\n%s", self.kind, len(batch), ex, traceback.format_exc())
            if len(batch) == 1:
                batch[0].error = ex
            else:
                for r in batch:
                    self._settle([r])

    def run(self):
        while not self._halt.is_set() or self.held:
            batch = self._next_batch()
            if batch is None:
                break
            t0 = time.time()
            self._settle(batch)
            self.batches.append(len(batch))
            log.info("%s batch of %d done in %.1f ms (queued %.1f ms)", self.kind, len(batch), (time.time() - t0) * 1e3,
                     (t0 - batch[0].t_in) * 1e3)
            for r in batch:
                r.done.set()


def chat_scheduler(pipeline, n_slots, prefix_cache=False, prefill_chunk=None):
    from .batching import SlotScheduler
    return SlotScheduler(pipeline.emu_model, n_slots, prefix_cache=prefix_cache, prefill_chunk=prefill_chunk)


def chunked_chat_scheduler(prefix_cache, prefill_chunk):
    """a make_scheduler for chat with chunked prefill (and prefix caching if asked)"""
    return lambda pipeline, n_slots: chat_scheduler(pipeline, n_slots, prefix_cache=prefix_cache, prefill_chunk=prefill_chunk)


def chat_prefix_scheduler(pipeline, n_slots):
    return chat_scheduler(pipeline, n_slots, prefix_cache=True)


def chat_slot_request(pipeline, inputs, knobs):
    from .batching import chat_request
    return chat_request(pipeline, inputs, **knobs)


def chat_prefix_request(pipeline, inputs, knobs):
    """a chat request with the keys a prefix-caching scheduler matches on"""
    from .batching import chat_request
    return chat_request(pipeline, inputs, prefix_keys=True, **knobs)


def generate_scheduler_for(pipeline, n_slots, encode_steps=None):
    """latent slots at the size the demo form always gets: forward's default 1024x1024"""
    from .batching import DenoiseSlotScheduler
    return DenoiseSlotScheduler(pipeline, n_slots or 4, encode_steps=encode_steps)


def encoding_generate_scheduler(encode_steps):
    """a make_scheduler for image generation whose prompts are encoded in regression slots, encode_steps per UNet step"""
    return lambda pipeline, n_slots: generate_scheduler_for(pipeline, n_slots, encode_steps=encode_steps)


def generate_slot_request(pipeline, inputs, knobs):
    from .batching import ImageRequest
    return ImageRequest(inputs=inputs, **knobs)


class ContinuousWorker(threading.Thread):
    """One pipeline under continuous batching: its thread owns the pipeline's engine and loops the scheduler's step() while
    anything is live or queued, and blocks on the queue when idle.  Same submit / stop surface as BatchingWorker.  A request
    that fails (prompt assembly, encoding, selection) answers with its own error and frees its slots; the others continue.
    `make_scheduler(pipeline, n_slots)` builds the scheduler it drives (default: chat's SlotScheduler; generate_scheduler
    for image generation) and `make_request(pipeline, inputs, knobs)` turns a submitted request into that scheduler's work
    (default: batching.chat_request).  `n_slots`: the scheduler's slots (chat default: the engine's llm_max_batch)."""

    def __init__(self, pipeline, n_slots=None, name=None, make_request=None, make_scheduler=None, kind="chat"):
        super().__init__(daemon=True, name=name or "emu-%s-continuous" % kind)
        self.pipeline, self.n_slots = pipeline, n_slots
        self.make_request = make_request or chat_slot_request
        self.make_scheduler = make_scheduler or chat_scheduler
        self.kind = kind
        self.q = queue.Queue()
        self.scheduler = None
        self._halt = threading.Event()

    def start(self):
        """build the scheduler before the thread starts: an engine that cannot run it (EMU_KV_COPY=1, tensor parallel) fails
        here, in the caller, instead of leaving a dead worker behind a queue"""
        self.scheduler = self.make_scheduler(self.pipeline, self.n_slots)
        super().start()

    def load(self):
        """queued + waiting for slots + running"""
        return self.q.qsize() + (self.scheduler.load() if self.scheduler is not None else 0)

    def submit(self, inputs, knobs, log_id="", timeout=None):
        r = _Request(inputs, knobs, log_id)
        self.q.put(r)
        if not r.done.wait(timeout):
            raise TimeoutError("request %s timed out" % log_id)
        if r.error is not None:
            raise r.error
        return r.result

    def stop(self):
        self._halt.set()
        self.q.put(None)

    def _admit(self, r):
        def answer(sr, r=r):
            r.result, r.error = sr.result, sr.error
            log.info("%s: %s done in %.1f ms", r.log_id, self.kind, (time.time() - r.t_in) * 1e3)
            r.done.set()
        try:
            sr = self.make_request(self.pipeline, r.inputs, r.knobs)
            sr.on_done, sr.tag = answer, r.log_id
            self.scheduler.submit(sr)
        except Exception as ex:  # the request fails, the server lives
            log.error("%s: %s request refused: %s\n%s", r.log_id, self.kind, ex, traceback.format_exc())
            r.error = ex
            r.done.set()

    def run(self):
        while True:
            idle = not self.scheduler.busy()
            if idle and self._halt.is_set():
                break
            try:
                r = self.q.get(block=idle)
                while True:
                    if r is None:
                        self._halt.set()
                    else:
                        self._admit(r)
                    r = self.q.get_nowait()
            except queue.Empty:
                pass
            if self.scheduler.busy():
                try:
                    self.scheduler.step()
                except Exception as ex:
                    log.error("continuous batching step failed: %s\n%s", ex, traceback.format_exc())
                    self.scheduler.abort(ex)


# ---- the form encoding of the demo front end (Emu2/demo/frontend/libs/chat_frontend.py:96-127) ----
def parse_form(content_type, body):
    """-> (fields: {name: str}, files: {name: bytes}) for multipart/form-data (what `requests.post(files=..., data=...)` sends
    when there are pictures) and application/x-www-form-urlencoded (what it sends when there are none)."""
    ctype = (content_type or "").lower()
    fields, files = {}, {}
    if ctype.startswith("multipart/form-data"):
        msg = BytesParser().parsebytes(b"Content-Type: " + content_type.encode() + b"\r\nMIME-Version: 1.0\r\n\r\n" + body)
        for part in msg.get_payload():
            name = part.get_param("name", header="content-disposition")
            if name is None:
                continue
            data = part.get_payload(decode=True)
            if part.get_filename() is not None:
                files[name] = data
            else:
                fields[name] = data.decode(part.get_content_charset() or "utf-8")
    else:
        for k, v in parse_qs(body.decode("utf-8"), keep_blank_values=True).items():
            fields[k] = v[-1]
    return fields, files


def decode_prompt(fields, files):
    """the interleaved `inputs` list the pipelines take: strings and PIL images in prompt order (backend.py:116-123)"""
    from PIL import Image
    inputs = []
    for kind, payload in json.loads(fields.get("prompt", "") or "[]"):
        if kind == "TEXT":
            inputs.append(payload)
        else:
            if payload not in files:
                raise KeyError("prompt refers to picture %r but no such file was uploaded" % payload)
            inputs.append(Image.open(io.BytesIO(files[payload])).convert("RGB"))
    return inputs


def chat_knobs(fields):
    """form fields -> EmuChatGeneration.forward keyword arguments with the reference's defaults and casts (backend.py:187-194)"""
    d = CHAT_DEFAULTS
    return dict(do_sample=str(fields.get("do_sample", "False")).lower() == "true",
                max_new_tokens=int(fields.get("max_new_tokens", d["max_new_tokens"])),
                temperature=float(fields.get("temperature", d["temperature"])),
                top_k=int(fields.get("top_k", d["top_k"])), top_p=float(fields.get("top_p", d["top_p"])),
                length_penalty=float(fields.get("length_penalty", d["length_penalty"])),
                num_beams=int(fields.get("num_beams", d["num_beams"])),
                repetition_penalty=float(fields.get("repetition_penalty", d["repetition_penalty"])))


def generation_knobs(fields):
    """EmuVisualGeneration.forward keyword arguments (backend.py:125-126,134); both fields are required, as in the reference"""
    return dict(guidance_scale=float(fields["classifier_free_guidance"]), num_inference_steps=int(fields["steps"]))


def image_to_webp_b64(image):
    buf = io.BytesIO()
    image.save(buf, format="WEBP")
    return base64.b64encode(buf.getvalue()).decode("ascii")


class EmuServer:
    """HTTP front + one worker per pipeline.  `chat` / `generate`: a pipeline or a list of pipelines (the reference's
    --chat-concurrency / --generate-concurrency instances); requests go to the worker with the shortest queue.
    `chat_scheduler` / `generate_scheduler`: "batching" (BatchingWorker, the default) or "continuous" (ContinuousWorker; for
    generation with max_images_per_batch latent slots).  `generate_encode_steps`: with continuous generation, encode the
    newcomers' prompts in regression slots, at most this many regression steps between two UNet steps."""

    def __init__(self, chat=None, generate=None, host="0.0.0.0", port=9000, max_wait_ms=0.0, max_images_per_batch=4,
                 cache_dir=None, announce=None, max_body_bytes=256 << 20, chat_scheduler="batching",
                 generate_scheduler="batching", chat_prefix_cache=False, chat_prefill_chunk=None,
                 generate_encode_steps=None):
        self.cache_dir = cache_dir
        self.chat_prefix_cache = bool(chat_prefix_cache)
        if self.chat_prefix_cache and chat_scheduler != "continuous":
            raise ValueError("chat_prefix_cache keeps KV-cache slots between requests: it needs chat_scheduler='continuous'")
        self.chat_prefill_chunk = None if chat_prefill_chunk is None else int(chat_prefill_chunk)
        if self.chat_prefill_chunk is not None and chat_scheduler != "continuous":
            raise ValueError("chat_prefill_chunk prefills newcomers inside the live slots' decode steps: it needs "
                             "chat_scheduler='continuous'")
        if self.chat_prefill_chunk is not None and self.chat_prefill_chunk < 1:
            raise ValueError("chat_prefill_chunk must be >= 1, got %d" % self.chat_prefill_chunk)
        self.generate_encode_steps = None if generate_encode_steps is None else int(generate_encode_steps)
        if self.generate_encode_steps is not None and generate_scheduler != "continuous":
            raise ValueError("generate_encode_steps interleaves prompt encoding with the UNet steps of live requests: it needs "
                             "generate_scheduler='continuous'")
        if self.generate_encode_steps is not None and self.generate_encode_steps < 1:
            raise ValueError("generate_encode_steps must be >= 1, got %d" % self.generate_encode_steps)
        self.max_body_bytes = int(max_body_bytes)
        if cache_dir:
            os.makedirs(cache_dir, exist_ok=True)

        def as_list(p):
            return [] if p is None else (list(p) if isinstance(p, (list, tuple)) else [p])

        def chat_cap(pipe):
            fn = getattr(pipe, "max_requests_per_batch", None)
            return (lambda knobs: fn(knobs.get("num_beams", 1))) if fn else (lambda knobs: 1)
        if chat_scheduler == "continuous":
            if announce is not None:
                raise ValueError("continuous batching runs on one GPU: it cannot follow a tensor-parallel instance")
            make_scheduler = chat_prefix_scheduler if self.chat_prefix_cache else None
            if self.chat_prefill_chunk is not None:
                make_scheduler = chunked_chat_scheduler(self.chat_prefix_cache, self.chat_prefill_chunk)
            self.chat_workers = [ContinuousWorker(p, name="emu-chat-%d" % i, make_scheduler=make_scheduler,
                                                  make_request=chat_prefix_request if self.chat_prefix_cache else None)
                                 for i, p in enumerate(as_list(chat))]
        elif chat_scheduler == "batching":
            self.chat_workers = [BatchingWorker(p, "chat", chat_cap(p), max_wait_ms, announce, "emu-chat-%d" % i)
                                 for i, p in enumerate(as_list(chat))]
        else:
            raise ValueError("chat_scheduler must be 'batching' or 'continuous', got %r" % (chat_scheduler,))
        # (no announce for generation: the UNet is not tensor parallel, follower ranks hold no generation pipeline)
        if generate_scheduler == "continuous":
            make_gen = (generate_scheduler_for if self.generate_encode_steps is None
                        else encoding_generate_scheduler(self.generate_encode_steps))
            self.gen_workers = [ContinuousWorker(p, max_images_per_batch, "emu-gen-%d" % i, generate_slot_request,
                                                 make_gen, "generate")
                                for i, p in enumerate(as_list(generate))]
        elif generate_scheduler == "batching":
            self.gen_workers = [BatchingWorker(p, "generate", (lambda knobs: max_images_per_batch)
                                               if hasattr(p, "forward_batch") else None, max_wait_ms, None, "emu-gen-%d" % i)
                                for i, p in enumerate(as_list(generate))]
        else:
            raise ValueError("generate_scheduler must be 'batching' or 'continuous', got %r" % (generate_scheduler,))
        server = self

        class Handler(BaseHTTPRequestHandler):
            protocol_version = "HTTP/1.1"

            def log_message(self, fmt, *a):
                log.debug("%s - " + fmt, self.address_string(), *a)

            def do_POST(self):
                n = int(self.headers.get("Content-Length") or 0)
                if n > server.max_body_bytes:          # a prompt is a few pictures: refuse to buffer anything absurd
                    self.send_error(413, "request body of %d bytes exceeds the limit of %d" % (n, server.max_body_bytes))
                    return
                body = self.rfile.read(n) if n else b""
                route = {"/v1/mmc": server.handle_chat, "/v1/mmg": server.handle_generate}.get(self.path.split("?")[0])
                if route is None:
                    self.send_error(404, "unknown route %s" % self.path)
                    return
                out = json.dumps(route(self.headers.get("Content-Type"), body)).encode()
                self.send_response(200)
                self.send_header("Content-Type", "application/json")
                self.send_header("Content-Length", str(len(out)))
                self.end_headers()
                self.wfile.write(out)

        self.httpd = ThreadingHTTPServer((host, port), Handler)
        self.httpd.daemon_threads = True
        self.port = self.httpd.server_address[1]

    # ---- the two routes; a failing request answers code -1 with the message, like the reference ----
    def _pick(self, workers, what, inputs=None):
        """the least loaded worker; with chat prefix caching, the worker holding the longest kept prefix of the prompt"""
        if not workers:
            raise RuntimeError("%s is disabled on this server" % what)
        if inputs is not None and self.chat_prefix_cache and len(workers) > 1:
            from .batching import prompt_signature
            sig = prompt_signature(inputs)
            held = [w.scheduler.cached_prefix(sig) if w.scheduler is not None else 0 for w in workers]
            if max(held) > 0:
                return min((w for w, n in zip(workers, held) if n == max(held)), key=lambda w: w.load())
        return min(workers, key=lambda w: w.load())

    def _save(self, log_id, name, image):
        if self.cache_dir:
            image.save(osp.join(self.cache_dir, "%s-%s.png" % (log_id, name)))

    def _answer(self, what, content_type, body, knobs_of, workers, finish):
        res, log_id, t0 = {"code": 0}, "", time.time()
        try:
            fields, files = parse_form(content_type, body)
            log_id = fields.get("log_id", "")
            log.info("%s: receive %s request", log_id, what)
            inputs = decode_prompt(fields, files)
            knobs = knobs_of(fields)
            log.info("%s: %s with hyper-parameters %s", log_id, what, knobs)
            res["data"] = finish(log_id, self._pick(workers, what, inputs if workers is self.chat_workers else None)
                                 .submit(inputs, knobs, log_id))
        except Exception as ex:
            log.error("%s: %s failed, err msg: %s\n%s", log_id, what, ex, traceback.format_exc())
            res = {"code": -1, "data": str(ex)}
        log.info("%s: %s complete with code %d, time: %.3fms", log_id, what, res["code"], (time.time() - t0) * 1e3)
        return res

    def handle_chat(self, content_type, body):
        return self._answer("chat", content_type, body, chat_knobs, self.chat_workers, lambda log_id, text: text)

    def handle_generate(self, content_type, body):
        def finish(log_id, out):
            image = out.image if hasattr(out, "image") else out
            self._save(log_id, "[RESULT]", image)
            return image_to_webp_b64(image)
        return self._answer("generation", content_type, body, generation_knobs, self.gen_workers, finish)

    # ---- life cycle ----
    def start(self):
        for w in self.chat_workers + self.gen_workers:
            w.start()
        self._thread = threading.Thread(target=self.httpd.serve_forever, daemon=True, name="emu-http")
        self._thread.start()
        return self

    def serve_forever(self):
        for w in self.chat_workers + self.gen_workers:
            w.start()
        self.httpd.serve_forever()

    def shutdown(self):
        self.httpd.shutdown()
        self.httpd.server_close()
        for w in self.chat_workers + self.gen_workers:
            w.stop()


# ---- tensor parallel: rank 0 serves, the other ranks follow ----
def make_announce(group=None):
    """-> announce(kind, batch_inputs, knobs) for rank 0: one broadcast of the admitted batch to every follower rank"""
    import torch.distributed as dist

    def announce(kind, batch_inputs, knobs):
        dist.broadcast_object_list([(kind, batch_inputs, knobs)], src=0, group=group)
    return announce


def follow(pipelines, group=None):
    """Ranks > 0 of a tensor-parallel instance: run every batch rank 0 admits (same calls, same order — the engine's collectives
    pair up), discard the outputs.  `pipelines`: {"chat": ..., "generate": ...}.  Returns when rank 0 broadcasts None."""
    import torch.distributed as dist
    while True:
        box = [None]
        dist.broadcast_object_list(box, src=0, group=group)
        if box[0] is None:
            return
        kind, batch_inputs, knobs = box[0]
        pipe = pipelines[kind]
        try:
            if len(batch_inputs) > 1 and hasattr(pipe, "forward_batch"):
                pipe.forward_batch(batch_inputs, **knobs)
            else:
                for i in batch_inputs:
                    pipe(inputs=i, **knobs)
        except Exception as ex:  # rank 0 reports the failure to the client; a follower only has to stay in step
            log.error("follower: %s batch failed: %s", kind, ex)


def release_followers(group=None):
    import torch.distributed as dist
    dist.broadcast_object_list([None], src=0, group=group)


def main(argv=None):
    ap = argparse.ArgumentParser(description="Emu2 demo back end (HTTP contract of Emu2/demo/backend/pytorch_model/backend.py) "
                                             "on the H100 engine")
    ap.add_argument("--port", type=int, default=9000)
    ap.add_argument("--host", type=str, default="0.0.0.0")
    ap.add_argument("--start-card", type=int, default=0)
    ap.add_argument("--disable-chat", action="store_true")
    ap.add_argument("--chat-concurrency", type=int, default=1)
    ap.add_argument("--chat-gpu-per-instance", type=int, default=1)
    ap.add_argument("--disable-generate", action="store_true")
    ap.add_argument("--generate-concurrency", type=int, default=1)
    ap.add_argument("--generate-gpu-per-instance", type=int, default=1)
    ap.add_argument("--model-path", type=str, default="./weight")
    ap.add_argument("--chat-max-rows", type=int, default=20, help="KV-cache rows of the chat engine (requests x num_beams)")
    ap.add_argument("--max-wait-ms", type=float, default=2.0)
    ap.add_argument("--max-images-per-batch", type=int, default=4)
    ap.add_argument("--continuous-batching", action="store_true",
                    help="chat requests join and leave the decode batch between steps (one GPU per chat instance)")
    ap.add_argument("--continuous-generation", action="store_true",
                    help="image requests join and leave the denoise batch between UNet steps, in --max-images-per-batch "
                         "latent slots")
    ap.add_argument("--prefix-cache", action="store_true",
                    help="with --continuous-batching: a finished chat request keeps its KV-cache slot, and a later turn of the "
                         "same conversation resumes from it and prefills only its new tokens")
    ap.add_argument("--prefill-chunk", type=int, default=None, metavar="C",
                    help="with --continuous-batching: a newcomer's prompt is prefilled in chunks of at most C tokens, each in "
                         "the same weight pass as the live requests' next token, so no live request waits for a whole prompt")
    ap.add_argument("--generate-encode-steps", type=int, default=None, metavar="R",
                    help="with --continuous-generation: newcomers' prompts are encoded together in LLaMA regression slots, "
                         "at most R regression steps between two UNet steps, so live requests never wait for a whole encode")
    ap.add_argument("--cache-dir", type=str, default="", help="keep request pictures / results here (the reference always does)")
    ap.add_argument("--safety-checker", action="store_true",
                    help="run the built-in NSFW safety checker (the checkpoint's safety_checker.* weights) on every generated "
                         "image: flagged images come back black, with nsfw_content_detected set")
    args = ap.parse_args(argv)
    if args.prefix_cache and not args.continuous_batching:
        ap.error("--prefix-cache keeps KV-cache slots between requests: it needs --continuous-batching")
    if args.prefill_chunk is not None and not args.continuous_batching:
        ap.error("--prefill-chunk prefills newcomers inside the live requests' decode steps: it needs --continuous-batching")
    if args.prefill_chunk is not None and args.prefill_chunk < 1:
        ap.error("--prefill-chunk must be >= 1")
    if args.generate_encode_steps is not None and not args.continuous_generation:
        ap.error("--generate-encode-steps interleaves prompt encoding with live requests' UNet steps: it needs "
                 "--continuous-generation")
    if args.generate_encode_steps is not None and args.generate_encode_steps < 1:
        ap.error("--generate-encode-steps must be >= 1")
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(name)s %(levelname)s %(message)s")
    import torch
    import torch.distributed as dist
    from .emu2.chat import EmuChatGeneration
    from .emu2.diffusion import EmuVisualGeneration
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    if max(args.chat_gpu_per_instance, args.generate_gpu_per_instance) > 1 and world == 1:
        ap.error("more than one GPU per instance = tensor parallelism: launch with torchrun, one process per GPU")
    if world > 1 and (args.chat_concurrency > 1 or args.generate_concurrency > 1):
        ap.error("under torchrun all ranks form ONE tensor-parallel instance; run more servers for more instances")
    if world > 1 and args.continuous_batching:
        ap.error("--continuous-batching runs on one GPU per chat instance: it is not available under torchrun")
    tp = {}
    if world > 1:
        # one tensor-parallel chat instance over all ranks: the library's communicator is created from an id made by rank 0
        import ctypes
        from . import _lib
        torch.cuda.set_device(args.start_card + int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
        buf = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            raw = ctypes.create_string_buffer(128)
            _lib.check(_lib.load().emu_nccl_unique_id(raw))
            buf.copy_(torch.frombuffer(bytearray(raw.raw), dtype=torch.uint8))
        dist.broadcast(buf, 0)
        tp = dict(tp_rank=rank, tp_size=world, nccl_uid=bytes(buf.cpu().numpy().tobytes()))
    device = args.start_card + (int(os.environ.get("LOCAL_RANK", "0")) if world > 1 else 0)
    chat, gen = [], []
    if not args.disable_generate and rank == 0:     # the UNet is not tensor parallel: generation lives on rank 0 only
        for i in range(args.generate_concurrency):
            torch.cuda.set_device(device)
            extra = {}
            if args.safety_checker:
                from .safety import SafetyChecker
                extra["safety_checker"] = SafetyChecker()
            gen.append(EmuVisualGeneration.from_pretrained(osp.join(args.model_path, "Emu2-Gen_pytorch_model.bf16.safetensors"),
                                                           dtype=torch.bfloat16, use_safetensors=True,
                                                           device="cuda:%d" % device, **extra))
            device += 1 if world == 1 else 0
    if not args.disable_chat:
        for i in range(args.chat_concurrency):
            torch.cuda.set_device(device)
            chat.append(EmuChatGeneration.from_pretrained(osp.join(args.model_path, "Emu2-Chat_pytorch_model.bf16.pth"),
                                                          instruct=True, dtype=torch.bfloat16, use_safetensors=False,
                                                          max_batch=args.chat_max_rows, device="cuda:%d" % device, **tp))
            device += 1 if world == 1 else 0
    if rank > 0:
        follow({"chat": chat[0] if chat else None})
        return
    srv = EmuServer(chat=chat, generate=gen, host=args.host, port=args.port, max_wait_ms=args.max_wait_ms,
                    max_images_per_batch=args.max_images_per_batch, cache_dir=args.cache_dir or None,
                    announce=make_announce() if world > 1 else None,
                    chat_scheduler="continuous" if args.continuous_batching else "batching",
                    generate_scheduler="continuous" if args.continuous_generation else "batching",
                    chat_prefix_cache=args.prefix_cache, chat_prefill_chunk=args.prefill_chunk,
                    generate_encode_steps=args.generate_encode_steps)
    log.info("serving on %s:%d (chat x%d, generate x%d)", args.host, srv.port, len(chat), len(gen))
    try:
        srv.serve_forever()
    finally:
        if world > 1:
            release_followers()


if __name__ == "__main__":
    main()
