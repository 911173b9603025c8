#!/usr/bin/env python
"""Trains the byte-level BPE tokenizer the benchmark's end-to-end leg runs with: Llama-3's tokenizer.json configuration (split regex,
ByteLevel pre-tokenizer, ignore_merges, the five control tokens) with an 8,192-entry vocabulary learned from a seeded corpus of what
OpsAgent actually sends — the reference's system prompts (tests/golden/prompts/*.txt), synthetic Pod manifests, kubectl tables, trivy
reports and ToolPrompt JSON.  No checkpoint tokenizer exists offline; with this one the verbatim prompts cost about as many tokens as
they would with a real Llama-3 vocabulary (analysisPrompt ~450, executeSystemPrompt_cn ~1,100 — the byte-level synthetic vocabulary
needs 1,965 / 3,233), so BASELINE's prompt lengths (P = 1536 / 1024 / 1280) hold the reference's real text.

    python tests/golden/gen_k8s_bpe.py     ->  tests/golden/bpe_k8s_8k.json   (needs the `tokenizers` library; the engine itself reads
                                               the JSON with its own C++ implementation, opsagent_b200/csrc/bpe.hpp)"""
import glob
import json
import os
import sys

from tokenizers import Regex, Tokenizer, decoders, models, pre_tokenizers, trainers

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from opsagent_b200.synthetic import copilot_tools          # noqa: E402
from opsagent_b200.workloads import EXECUTE_QUESTIONS, synthetic_pod_yaml   # noqa: E402

LLAMA3 = r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}{1,3}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|\s+(?!\S)|\s+"
SPECIALS = ["<|begin_of_text|>", "<|end_of_text|>", "<|start_header_id|>", "<|end_header_id|>", "<|eot_id|>"]


def corpus():
    """Domain text WITHOUT the four prompts the benchmark sends (a tokenizer trained on them would memorise whole sentences): the rest of
    the reference tree read at generation time (Go sources with their zh/en comments, README, configs — only the learned vocabulary is
    committed, no reference text), plus seeded synthetic manifests / kubectl / trivy / ToolPrompt JSON."""
    ref = os.environ.get("OA_REFERENCE", "")
    if not os.path.isdir(ref):
        sys.exit("set OA_REFERENCE to a checkout of the reference (myysophia/OpsAgent @ c1109da1)")
    held_out = [open(os.path.join(HERE, "prompts", n + ".txt"), encoding="utf-8").read()
                for n in ("executeSystemPrompt_cn", "diagnoseSystemPrompt", "analysisPrompt", "auditPrompt")]
    docs = []
    for root, _dirs, files in sorted(os.walk(ref)):
        for f in sorted(files):
            if f.endswith((".go", ".md", ".yaml", ".yml", ".json", ".sh")) or f == "Dockerfile":
                text = open(os.path.join(root, f), encoding="utf-8", errors="ignore").read()
                for h in held_out:
                    text = text.replace(h, "")
                docs.append(text)
    tools = copilot_tools(11)
    for i in range(200):
        docs.append(synthetic_pod_yaml(10_000 + i, 2500, seed=7))
    for i in range(80):
        docs.append(tools["kubectl"](f"get pods -n ns-{i} -o wide"))
        docs.append(tools["trivy"](f"registry.local/team{i % 30}/img{i}:1.{i}"))
        q = EXECUTE_QUESTIONS[i % len(EXECUTE_QUESTIONS)]
        docs.append(json.dumps({"question": q, "thought": "I should list the resources with kubectl and inspect their status", "action":
                                {"name": "kubectl", "input": f"get pods -n ns-{i} --no-headers"}, "observation": "", "final_answer": ""}, ensure_ascii=False))
    return docs


def main():
    tok = Tokenizer(models.BPE(ignore_merges=True))
    tok.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(LLAMA3), behavior="isolated", invert=False),
                                                 pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=8192, special_tokens=SPECIALS, initial_alphabet=pre_tokenizers.ByteLevel.alphabet(), show_progress=False)
    tok.train_from_iterator(corpus(), trainer)
    out = os.path.join(HERE, "bpe_k8s_8k.json")
    tok.save(out, pretty=False)
    for name in ("analysisPrompt", "diagnoseSystemPrompt", "executeSystemPrompt_cn", "auditPrompt"):
        text = open(os.path.join(HERE, "prompts", name + ".txt"), encoding="utf-8").read()
        print(f"{name:24s} {len(text.encode()):5d} bytes -> {len(tok.encode(text, add_special_tokens=False).ids):5d} tokens")
    print("vocab", tok.get_vocab_size(), "file", os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
