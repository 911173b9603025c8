"""The boundary is a C ABI: include/opsagent_b200.h must compile as plain C99 (no C++ types, no default arguments) and a C program
linked against the library must be able to drive it.  No compute calls: engine creation is only asked to reject a bad config."""
import os
import shutil
import subprocess
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "opsagent_b200", "lib")

SRC = textwrap.dedent(r'''
    #include <stdio.h>
    #include <string.h>
    #include "opsagent_b200.h"

    int main(int argc, char** argv) {
        oa_engine* e = (oa_engine*)0;
        int rc = oa_engine_create("{\"model\": \"no-such-model\"}", &e);
        if (rc != 400 || e != (oa_engine*)0) { printf("create rc=%d\n", rc); return 1; }
        if (!strstr(oa_last_error(), "unknown model")) { printf("error text: %s\n", oa_last_error()); return 2; }
        if (!strstr(oa_version(), "sm_90a")) return 3;
        {   /* request struct is plain data */
            oa_msg m[2]; oa_chat_req r; oa_chat_resp out;
            memset(&r, 0, sizeof r); memset(&out, 0, sizeof out);
            m[0].role = "system"; m[0].content = "s"; m[1].role = "user"; m[1].content = "u";
            r.model = "m"; r.msgs = m; r.n_msgs = 2; r.max_tokens = 8; r.temperature = 0.0f; r.flags = OA_FLAG_IGNORE_EOS;
            if (oa_chat_complete((oa_engine*)0, &r, &out) != 400) return 4;      /* null engine is a bad request, not a crash */
        }
        if (argc > 1) {      /* byte-level BPE through the C ABI */
            int32_t ids[64]; int32_t n = 0; char buf[64]; int32_t nb = 0;
            if (oa_host_bpe_encode(argv[1], "kubectl get pods", 16, ids, 64, &n) != 0 || n <= 0) { printf("encode: %s\n", oa_last_error()); return 5; }
            if (oa_host_bpe_decode(argv[1], ids, n, buf, 64, &nb) != 0 || nb != 16 || memcmp(buf, "kubectl get pods", 16)) return 6;
        }
        printf("ok\n");
        return 0;
    }
''')


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_header_is_c99_and_a_c_program_links_and_runs(tmp_path):
    if not os.path.exists(os.path.join(LIBDIR, "libopsagent_b200.so")):
        pytest.skip("library not built")
    src = tmp_path / "abi.c"; src.write_text(SRC)
    exe = tmp_path / "abi"
    cmd = ["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
           "-L", LIBDIR, "-lopsagent_b200", f"-Wl,-rpath,{LIBDIR}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    tok = os.path.join(ROOT, "tests", "golden", "bpe_llama3_tiny.json")
    r = subprocess.run([str(exe), tok], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout, r.stderr)


SRC_GPU = textwrap.dedent(r'''
    #include <stdio.h>
    #include <string.h>
    #include "opsagent_b200.h"

    /* a strict-C99 caller doing real work on the GPU: create an engine, submit a chat completion with the error-buffer variants
       (what the cgo binding uses), wait with a timeout, print the generated token ids; then cancel a second request */
    int main(int argc, char** argv) {
        oa_engine* e = (oa_engine*)0; oa_msg m[2]; oa_chat_req r; oa_chat_resp out; uint64_t t = 0, t2 = 0; char err[256]; int rc, i, spins = 0; char st[2048];
        if (argc < 2) return 9;
        rc = oa_engine_create(argv[1], &e);
        if (rc != 0) { printf("create: %d %s\n", rc, oa_last_error()); return 1; }
        memset(&r, 0, sizeof r); memset(&out, 0, sizeof out);
        m[0].role = "system"; m[0].content = "You are a Kubernetes expert."; m[1].role = "user"; m[1].content = "how many namespace in the cluster?";
        r.model = ""; r.msgs = m; r.n_msgs = 2; r.max_tokens = 16; r.temperature = 0.0f; r.flags = OA_FLAG_IGNORE_EOS;
        rc = oa_chat_submit_ex(e, &r, &t, err, sizeof err);
        if (rc != 0) { printf("submit: %d %s\n", rc, err); return 2; }
        do { rc = oa_chat_wait_ex(e, t, 50, &out, err, sizeof err); ++spins; } while (rc == 408 && spins < 2000);
        if (rc != 0) { printf("wait: %d %s\n", rc, err); return 3; }
        printf("ids:");
        for (i = 0; i < out.completion_tokens; ++i) printf(" %d", (int)out.token_ids[i]);
        printf("\nprompt_tokens: %d\n", (int)out.prompt_tokens);
        oa_free_resp(&out);
        r.max_tokens = 400;
        if (oa_chat_submit_ex(e, &r, &t2, err, sizeof err) != 0) return 4;
        if (oa_chat_cancel(e, t2) != 0) return 5;
        if (oa_chat_wait_ex(e, t2, 10, &out, err, sizeof err) != 400 || !strstr(err, "unknown ticket")) { printf("after cancel: %s\n", err); return 6; }
        r.model = "not-this-model";
        if (oa_chat_submit_ex(e, &r, &t2, err, sizeof err) != 400 || !strstr(err, "is not loaded")) { printf("alias: %s\n", err); return 7; }
        if (oa_engine_stats(e, st, sizeof st) != 0 || !strstr(st, "\"cancelled\": 1")) { printf("stats: %s\n", st); return 8; }
        oa_engine_destroy(e);
        printf("ok\n");
        return 0;
    }
''')


@pytest.mark.gpu
@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_c_program_runs_a_chat_completion_on_the_gpu_and_matches_the_oracle(tmp_path):
    """the boundary driven from strict C99 with real compute: the ids the C caller gets back equal the oracle's greedy decode"""
    import json
    import numpy as np
    from oracle import oracle as O          # checker only
    spec = O.PRESETS["tiny-llama"]
    cfg = spec.engine_json(num_pages=32, max_seq_len=512, max_batch=4, max_step_tokens=256)
    src = tmp_path / "abi_gpu.c"; src.write_text(SRC_GPU)
    exe = tmp_path / "abi_gpu"
    cmd = ["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
           "-L", LIBDIR, "-lopsagent_b200", f"-Wl,-rpath,{LIBDIR}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), json.dumps(cfg)], capture_output=True, text=True, timeout=240)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), (r.returncode, r.stdout, r.stderr)
    got = [int(x) for x in r.stdout.split("ids:")[1].split("\n")[0].split()]
    ids = O.apply_chat_template(spec, [("system", "You are a Kubernetes expert."), ("user", "how many namespace in the cluster?")])
    assert int(r.stdout.split("prompt_tokens:")[1].split()[0]) == len(ids)
    orc = O.Oracle(spec, max_pos=512, mode=1)
    ref, margins, _ = orc.generate(np.array(ids, np.int32), 16)
    orc.close()
    k = 0
    while k < 16 and got[k] == ref[k]:
        k += 1
    assert len(got) == 16 and (k == 16 or margins[k] <= 5e-2), (k, got, list(ref))


def _build_server(tmp_path):
    exe = tmp_path / "opsagent_serve"
    cmd = ["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-O2", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "integration", "c", "opsagent_serve.c"),
           "-o", str(exe), "-L", LIBDIR, "-lopsagent_b200", f"-Wl,-rpath,{LIBDIR}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_standalone_c_server_builds_and_fails_loudly_without_a_gpu(tmp_path):
    """integration/c/opsagent_serve.c: strict C99 on the C ABI only.  Without CUDA it must say so and exit 1 — never serve from a CPU path."""
    import torch
    exe = _build_server(tmp_path)
    r = subprocess.run([str(exe), "--bogus"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2 and "usage:" in r.stderr
    r = subprocess.run([str(exe), "--engine", "[]"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 2
    if torch.cuda.is_available():
        pytest.skip("the no-GPU half of this check is for the GPU-less container")
    r = subprocess.run([str(exe), "--engine", '{"model": "llama-3.2-1b"}', "--port", "0"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "no CUDA device" in r.stderr and "no CPU fallback" in r.stderr


@pytest.mark.gpu
@pytest.mark.skipif(shutil.which("gcc") is None, reason="no C compiler")
def test_standalone_c_server_serves_chat_completions_on_the_gpu(tmp_path):
    """the C server with two replicas of a tiny model on this GPU: the wire answer equals the engine's own greedy completion; SIGTERM exits 0"""
    import http.client
    import json
    import signal
    from oracle import oracle as O          # presets only
    from opsagent_b200 import Engine
    spec = O.PRESETS["tiny-llama"]
    cfg = spec.engine_json(num_pages=64, max_seq_len=512, max_batch=4, max_step_tokens=256)
    exe = _build_server(tmp_path)
    p = subprocess.Popen([str(exe), "--engine", json.dumps(cfg), "--devices", "0,0", "--port", "0", "--api-key", "k"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    try:
        line = json.loads(p.stdout.readline())
        assert line["replicas"] == 2
        port = int(line["listening"].rsplit(":", 1)[1].split("/")[0])
        msgs = [("system", "You are a Kubernetes expert."), ("user", "how many namespace in the cluster?")]
        c = http.client.HTTPConnection("127.0.0.1", port, timeout=120)
        c.request("POST", "/v1/chat/completions", body=json.dumps({"model": "gpt-4", "max_tokens": 12, "messages": [{"role": r, "content": t} for r, t in msgs]}),
                  headers={"Authorization": "Bearer k"})
        r = c.getresponse(); d = json.loads(r.read())
        assert r.status == 200, d                     # "gpt-4": the server answers to any model name (execute.go:168-171 sends it when currentModel is empty)
        c.request("POST", "/v1/chat/completions", body="{}", headers={"Authorization": "Bearer wrong"})
        r = c.getresponse(); r.read()
        assert r.status == 401
        eng = Engine(cfg)
        ref = eng.chat_complete(spec.name, msgs, 12)
        eng.close()
        assert d["choices"][0]["message"]["content"] == bytes(ref.content).decode("utf-8", "replace").rstrip("\n")
        assert d["usage"]["completion_tokens"] == ref.completion_tokens
    finally:
        p.send_signal(signal.SIGTERM)
        try:
            rc = p.wait(timeout=60)
        except subprocess.TimeoutExpired:
            p.kill(); rc = -9
    assert rc == 0, p.stderr.read()[-500:]
