"""tools/time_multi_context.py -- 7B q4_0 greedy decode with one context and with two live contexts that take turns.

Uses bench.py's synthetic LLaMA-7B q4_0 file (written once, to $FASTLLAMA_BENCH_DIR or /tmp, unless --model is given).  Every context
ingests the same prompt and runs one warm-up token (its decode plan is built and its graph captured there), then the timed part generates
--tokens tokens per context:
  - one:       one context, generate calls of --chunk tokens, then its KV cache reset, the prompt ingested again and the same again
               (so every configuration decodes each position range the same number of times);
  - per_call:  two contexts, alternating every generate call of --chunk tokens;
  - one_1, per_token: the same two with generate calls of one token (the per-call cost of the bridge is in both).
Prints one JSON line per configuration: wall-clock tokens/s and the plan builds / graph captures the timed part added
(ggml_b200_get_contexts), which should be 0.  Asserts nothing about speed.

    python tools/time_multi_context.py [--model PATH] [--tokens 384] [--chunk 16] [--mmap]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PROMPT = "Two conversations share one GPU and take turns."
GREEDY = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)


class _Contexts(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("live_states", "plan_builds", "graph_captures", "external_copies", "external_mappings", "external_bytes")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default=None)
    ap.add_argument("--tokens", type=int, default=384, help="tokens per context in the timed part (n_ctx is 512)")
    ap.add_argument("--chunk", type=int, default=16, help="tokens per generate call in 'one' and 'per_call'")
    ap.add_argument("--mmap", action="store_true", help="load with use_mmap (the two contexts share one device copy of the weights)")
    args = ap.parse_args()

    import bench
    from fastllama_b200.build import lib_path
    from fastllama_b200.model import Model, QuietLogger

    path = args.model or bench.ensure_model("7B", "q4_0")
    lib = lib_path("pyfastllama.so")
    g = C.CDLL(lib)

    def counters():
        if not hasattr(g, "ggml_b200_get_contexts"):          # a build from before per-context decode states
            return None, None
        c = _Contexts()
        g.ggml_b200_get_contexts(C.byref(c))
        return int(c.plan_builds), int(c.graph_captures)

    def load():
        m = Model(path, num_threads=1, n_ctx=512, n_batch=16, last_n_size=64, use_mmap=args.mmap, logger=QuietLogger(), library_path=lib)
        assert m.ingest(PROMPT)
        assert m.generate(lambda s: None, num_tokens=1, **GREEDY)        # builds the plan and captures the graph
        return m

    def gen(m, n):
        assert m.generate(lambda s: None, num_tokens=n, **GREEDY)

    def restart(m):
        assert m.reset() and m.ingest(PROMPT)
        gen(m, 1)

    def report(name, tokens, seconds, c0):
        c1 = counters()
        print(json.dumps({"config": name, "tokens": tokens, "tokens_per_s": round(tokens / seconds, 2), "seconds": round(seconds, 3),
                          "plan_builds_added": None if c1[0] is None else c1[0] - c0[0],
                          "graph_captures_added": None if c1[1] is None else c1[1] - c0[1], "decode_mode": int(g.ggml_b200_decode_mode()),
                          "mmap": args.mmap}), flush=True)

    a = load()
    b = load()
    for chunk, one_name, two_name in ((args.chunk, "one", "per_call"), (1, "one_1", "per_token")):
        restart(a)
        restart(b)
        c0 = counters()
        t = 0.0
        for rnd in range(2):                      # context a twice over the same positions
            if rnd:
                restart(a)
            t0 = time.perf_counter()
            for _ in range(args.tokens // chunk):
                gen(a, chunk)
            t += time.perf_counter() - t0
        report(one_name, 2 * (args.tokens // chunk) * chunk, t, c0)
        restart(a)
        c0 = counters()
        t0 = time.perf_counter()
        for _ in range(args.tokens // chunk):
            gen(a, chunk)
            gen(b, chunk)
        report(two_name, 2 * (args.tokens // chunk) * chunk, time.perf_counter() - t0, c0)
    a.close()
    b.close()


if __name__ == "__main__":
    main()
