"""Measure grammar-constrained generation on one GPU: a seeded byte-level vocabulary of 151 936 tokens and the Qwen3
decoder with seeded weights at the 8B or 4B shape (``tools/bench_llm.py``'s ``make_plan``).

Reports, for each of the function-calling protocol's grammars (the decision, the follow-up and the arguments of
``search_knowledge_base``): its DFA states, the host compile time and the device token index build time; the sampler's
time per step masked against unmasked (CUDA events); and decode ms/token (forward + sampling) at context 1k with and
without a grammar.  The card's name and power limit are read in the same process; prints one JSON line.

    python tools/bench_grammar.py [--model 8b|4b|both] [--steps 64]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_llm import SHAPES, make_plan  # noqa: E402

from raglite_b200._grammar import compile_gbnf, json_schema_to_gbnf  # noqa: E402
from raglite_b200._llm import LlmEngine  # noqa: E402
from raglite_b200._rag import SEARCH_KNOWLEDGE_BASE_TOOL  # noqa: E402
from raglite_b200._tools import DECISION_GRAMMAR, FOLLOW_UP_GRAMMAR  # noqa: E402

NAMES = '"functions.search_knowledge_base:"'
GRAMMARS = {"decision": DECISION_GRAMMAR.format(names=NAMES), "follow_up": FOLLOW_UP_GRAMMAR.format(names=NAMES),
            "arguments": json_schema_to_gbnf(SEARCH_KNOWLEDGE_BASE_TOOL["function"]["parameters"])}


def synthetic_tokenizer(V: int, seed: int = 0) -> SimpleNamespace:
    """256 byte tokens, seeded pieces of 1 to 12 bytes (mostly printable), and the two end-of-generation tokens."""
    rng = np.random.default_rng(seed)
    pieces = [bytes([b]) for b in range(256)]
    lens = rng.integers(1, 13, V - 258)
    for n in lens:
        pieces.append(bytes(rng.integers(32, 127, int(n), dtype=np.uint8)) if rng.random() < 0.9
                      else bytes(rng.integers(0, 256, int(n), dtype=np.uint8)))
    pieces += [b"<|im_end|>", b"<|endoftext|>"]
    return SimpleNamespace(token_bytes=pieces, ids={"<|im_end|>": V - 2, "<|endoftext|>": V - 1})


def _events(fn, reps: int) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def bench(name: str, steps: int) -> dict:
    shape = SHAPES[name]
    eng = LlmEngine(make_plan(shape), synthetic_tokenizer(shape["vocab"]), n_ctx=1024 + steps + 2, prefill_chunk=512)
    out: dict = {"model": name, "vocab": shape["vocab"], "grammars": {}}
    eng.grammar_index('root ::= "x"')   # uploads the vocabulary's bytes once, outside the timed builds
    for g, text in GRAMMARS.items():
        t = time.perf_counter()
        dfa = compile_gbnf(text)
        compile_s = time.perf_counter() - t
        torch.cuda.synchronize()
        t = time.perf_counter()
        eng.grammar_index(dfa)
        torch.cuda.synchronize()
        out["grammars"][g] = {"states": dfa.n_states, "compile_ms": round(compile_s * 1e3, 1),
                              "index_build_ms": round((time.perf_counter() - t) * 1e3, 2),
                              "index_bytes": dfa.n_states * shape["vocab"] * 2}
    gi = eng.grammar_index(GRAMMARS["arguments"])
    rng = np.random.default_rng(1)
    eng.reset()
    eng.prefill(rng.integers(0, 256, 1024).tolist())
    hist = rng.integers(0, 256, 64).tolist()
    kw = dict(temperature=0.6, top_k=20, top_p=0.95, min_p=0.0, repeat_penalty=1.1, u=0.5)
    eng.grammar_state.zero_()
    out["sample_ms"] = {"unmasked": round(_events(lambda: eng.sample(hist, **kw), 200), 4),
                        "masked": round(_events(lambda: eng.sample(hist, grammar=gi, **kw), 200), 4)}
    decode = {}
    for label, g in (("unmasked", None), ("masked", gi)):
        eng.reset()
        eng.prefill(rng.integers(0, 256, 1024).tolist())
        eng.grammar_state.zero_()
        eng._tok.fill_(ord("{"))

        def step(g=g) -> None:
            eng._forward_dev(eng._tok.data_ptr(), 1)
            eng.sample(hist, grammar=g, **kw)

        decode[label] = round(_events(step, steps), 3)
    out["decode_ms_per_token_ctx1k"] = decode
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="8b", choices=["8b", "4b", "both"])
    ap.add_argument("--steps", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grammar needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=False).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else None,
           "models": [bench(m, a.steps) for m in (["8b", "4b"] if a.model == "both" else [a.model])]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
