#!/usr/bin/env python
"""Extracts the reference's system prompts VERBATIM into fixtures (contract text, SURVEY.md §8c: "the system prompts verbatim").

These strings are the bytes the reference feeds the Chat seam on every request, so tests and bench.py must tokenise exactly
them, not a paraphrase.  Run with a checkout of the reference (myysophia/OpsAgent @ c1109da1):

    OA_REFERENCE=<path to the reference checkout> python tests/golden/prompts/extract_prompts.py

Writes <name>.txt (raw UTF-8 bytes of the Go raw-string constant, no trailing newline added) and index.json
(name -> source file:line range, byte length, sha256).  tests/test_host_logic.py checks the fixtures against index.json.
"""
import hashlib
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("OA_REFERENCE", "")

# constant name -> (file, how the workload uses it)
SOURCES = {
    "executeSystemPrompt_cn": ("pkg/handlers/execute.go", "system message of POST /execute (execute.go:190-199) — BASELINE configs[0], configs[2] 'execute', configs[3]"),
    "diagnoseSystemPrompt": ("cmd/kube-copilot/diagnose.go", "system message of `kube-copilot diagnose` — configs[2] 'diagnose'"),
    "analysisPrompt": ("pkg/workflows/analyze.go", "instructions of the swarm analysis flow (analyze.go:47-75) — configs[1], configs[2] 'analyze'"),
    "auditPrompt": ("pkg/workflows/audit.go", "instructions of the swarm audit flow (audit.go:58-87) — configs[4]"),
    "generatePrompt": ("pkg/workflows/generate.go", "instructions of the swarm generate flow"),
    "assistantPrompt": ("pkg/workflows/assistant.go", "instructions of the swarm assistant flow"),
    "assistantPrompt_cn": ("pkg/workflows/assistant.go", "instructions of the swarm assistant flow (zh)"),
}
# one-line System strings of the swarm flows (SimpleFlow.System), extracted as Go interpreted-string literals
SYSTEM_LINES = {
    "analysisSystem": ("pkg/workflows/analyze.go", r'System:\s+"((?:[^"\\]|\\.)*)"'),
    "auditSystem": ("pkg/workflows/audit.go", r'System:\s+"((?:[^"\\]|\\.)*)"'),
}


def extract(ref_root=REF):
    out = {}
    for name, (rel, use) in SOURCES.items():
        src = open(os.path.join(ref_root, rel), encoding="utf-8").read()
        m = re.search(r"const\s+" + re.escape(name) + r"\s*=\s*`", src)
        if not m:
            raise SystemExit(f"{name} not found in {rel}")
        end = src.index("`", m.end())
        text = src[m.end():end]
        l0 = src.count("\n", 0, m.start()) + 1
        l1 = src.count("\n", 0, end) + 1
        out[name] = (text, f"{rel}:{l0}-{l1}", use)
    for name, (rel, pat) in SYSTEM_LINES.items():
        src = open(os.path.join(ref_root, rel), encoding="utf-8").read()
        m = re.search(pat, src)
        if not m:
            raise SystemExit(f"{name} not found in {rel}")
        text = json.loads('"' + m.group(1) + '"')          # Go interpreted string == JSON string for these ASCII lines
        line = src.count("\n", 0, m.start()) + 1
        out[name] = (text, f"{rel}:{line}", "SimpleFlow.System of the flow")
    return out


def main():
    ex = extract()
    index = {}
    for name, (text, where, use) in ex.items():
        raw = text.encode("utf-8")
        with open(os.path.join(HERE, name + ".txt"), "wb") as f:
            f.write(raw)
        index[name] = {"source": where, "bytes": len(raw), "sha256": hashlib.sha256(raw).hexdigest(), "use": use}
    with open(os.path.join(HERE, "index.json"), "w") as f:
        json.dump(index, f, indent=1, ensure_ascii=False)
        f.write("\n")
    for k, v in index.items():
        print(f"{k:26s} {v['bytes']:6d} B  {v['source']}")


if __name__ == "__main__":
    sys.exit(main())
