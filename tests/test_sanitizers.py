"""Host-side race / memory-error detection (SURVEY.md 5.2): the native HTTP front under TSAN and ASAN+UBSAN with a stub engine, and the parsers of
untrusted bytes (BPE, tokenizer.json, config JSON, safetensors headers, the ToolPrompt automaton + token masks) under ASAN+UBSAN.  The device side is
covered by compute-sanitizer on a GPU machine: tools/sanitize_gpu.sh."""
import pytest

# ---- race / memory-error detection on the host side (SURVEY.md 5.2) -----------------------------------------------------------------------
import os
import subprocess
import sys

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("sanitizer", ["thread", "address,undefined"])
def test_front_under_sanitizers_with_a_stub_engine(sanitizer, tmp_path):
    """tests/sanitize/front_harness.cpp: the front compiled with a stub engine under TSAN / ASAN+UBSAN, 24 concurrent clients incl. hostile ones,
    stopped with connections still open.  Any data race, heap error or UB makes the binary exit non-zero."""
    exe = tmp_path / "front_harness"
    cmd = ["g++", "-std=c++17", "-O1", "-g", f"-fsanitize={sanitizer}", "-fno-omit-frame-pointer", "-I", os.path.join(_ROOT, "opsagent_b200", "csrc"),
           os.path.join(_ROOT, "tests", "sanitize", "front_harness.cpp"), os.path.join(_ROOT, "opsagent_b200", "csrc", "http_server.cpp"), "-o", str(exe), "-lpthread"]
    b = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    if b.returncode != 0 and ("cannot find" in b.stderr or "unrecognized" in b.stderr):
        pytest.skip("sanitizer runtime not installed: " + b.stderr[-200:])
    assert b.returncode == 0, b.stderr[-2000:]
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0 exitcode=66", ASAN_OPTIONS="detect_leaks=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert "0 check failures" in r.stdout and "WARNING: ThreadSanitizer" not in r.stderr and "ERROR: AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr


def test_host_parsers_and_grammar_under_asan_ubsan(tmp_path):
    """tests/sanitize/host_fuzz.cpp: BPE on arbitrary bytes (round trip), damaged tokenizer.json / config JSON / safetensors headers, random legal
    walks of the ToolPrompt automaton with its token masks, hostile chat-template input — under ASAN + UBSAN; results or exceptions, no reports."""
    exe = tmp_path / "host_fuzz"
    b = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-I", os.path.join(_ROOT, "opsagent_b200", "csrc"),
                        os.path.join(_ROOT, "tests", "sanitize", "host_fuzz.cpp"), "-o", str(exe)], capture_output=True, text=True, timeout=600)
    if b.returncode != 0 and ("cannot find" in b.stderr or "unrecognized" in b.stderr):
        pytest.skip("sanitizer runtime not installed: " + b.stderr[-200:])
    assert b.returncode == 0, b.stderr[-2000:]
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    r = subprocess.run([str(exe), os.path.join(_ROOT, "tests", "golden", "bpe_k8s_8k.json"), str(tmp_path), "150"], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, (r.stdout[-500:], r.stderr[-3000:])
    assert r.stdout.startswith("ok:") and "AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
