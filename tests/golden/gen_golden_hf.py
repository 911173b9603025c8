"""Generate the golden fixtures that pin the CPU oracle against an INDEPENDENT implementation:
HF transformers LlamaForCausalLM / Qwen2ForCausalLM, fp32, CPU, greedy.

The reference (myysophia/OpsAgent) ships no model arithmetic and no golden vectors for this path
(SURVEY.md §8c), so these fixtures are the pin.  Run in the build container (needs transformers +
torch on CPU; does NOT need the reference):

    python tests/golden/gen_golden_hf.py [config ...]

Writes tests/golden/hf_<config>.npz with: prompt ids, HF fp32 logits for every prompt position,
HF greedy continuation and its per-step top1-top2 margins.  The weights are the oracle's own
deterministic tensors (seed -> bf16), loaded into the HF module as fp32.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

CASES = {"tiny-llama": dict(T=24, G=12, seed=7), "tiny-llama-d128": dict(T=20, G=10, seed=8),
         "tiny-qwen": dict(T=28, G=12, seed=9), "tiny-llama-g8": dict(T=22, G=10, seed=10), "tiny-llama-mha": dict(T=18, G=10, seed=11),
         "tiny-qwen-tp4": dict(T=20, G=10, seed=12), "tiny-llama-tp8": dict(T=20, G=10, seed=13), "tiny-llama-8bheads": dict(T=20, G=10, seed=14)}


def hf_model(spec: O.ModelSpec, orc: O.Oracle):
    import transformers
    common = dict(hidden_size=spec.hidden, intermediate_size=spec.ffn, num_hidden_layers=spec.n_layers,
                  num_attention_heads=spec.n_heads, num_key_value_heads=spec.n_kv_heads, head_dim=spec.head_dim,
                  vocab_size=spec.vocab, rms_norm_eps=spec.rms_eps, max_position_embeddings=131072,
                  tie_word_embeddings=bool(spec.tie_embeddings), attention_bias=False, hidden_act="silu")
    rope = {"rope_type": "default", "rope_theta": spec.rope_theta}
    if spec.rope_scaling == 1:
        rope = {"rope_type": "llama3", "rope_theta": spec.rope_theta, "factor": spec.rope_factor,
                "low_freq_factor": spec.rope_low_freq, "high_freq_factor": spec.rope_high_freq,
                "original_max_position_embeddings": spec.rope_orig_ctx}
    if spec.qkv_bias:
        common.pop("attention_bias")
        cfg = transformers.Qwen2Config(**common, rope_parameters=rope, use_sliding_window=False)
        model = transformers.Qwen2ForCausalLM(cfg)
    else:
        cfg = transformers.LlamaConfig(**common, rope_parameters=rope)
        model = transformers.LlamaForCausalLM(cfg)
    model = model.to(torch.float32).eval()
    H, qd, kd, F, V = spec.hidden, spec.n_heads * spec.head_dim, spec.n_kv_heads * spec.head_dim, spec.ffn, spec.vocab
    t = lambda layer, kind, shape: torch.from_numpy(orc.tensor_f32(layer, kind, shape).copy())
    sd = {"model.embed_tokens.weight": t(-1, 0, (V, H)), "model.norm.weight": t(-1, 1, (H,))}
    sd["lm_head.weight"] = sd["model.embed_tokens.weight"] if spec.tie_embeddings else t(-1, 2, (V, H))
    for l in range(spec.n_layers):
        p = f"model.layers.{l}."
        sd[p + "self_attn.q_proj.weight"] = t(l, "wq", (qd, H)); sd[p + "self_attn.k_proj.weight"] = t(l, "wk", (kd, H))
        sd[p + "self_attn.v_proj.weight"] = t(l, "wv", (kd, H)); sd[p + "self_attn.o_proj.weight"] = t(l, "wo", (H, qd))
        sd[p + "mlp.gate_proj.weight"] = t(l, "wg", (F, H)); sd[p + "mlp.up_proj.weight"] = t(l, "wu", (F, H))
        sd[p + "mlp.down_proj.weight"] = t(l, "wd", (H, F))
        sd[p + "input_layernorm.weight"] = t(l, "ln1", (H,)); sd[p + "post_attention_layernorm.weight"] = t(l, "ln2", (H,))
        if spec.qkv_bias:
            sd[p + "self_attn.q_proj.bias"] = t(l, "bq", (qd,)); sd[p + "self_attn.k_proj.bias"] = t(l, "bk", (kd,))
            sd[p + "self_attn.v_proj.bias"] = t(l, "bv", (kd,))
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "lm_head" in m for m in missing), missing
    return model


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    only = set(sys.argv[1:])               # optional: regenerate just the named configs
    for name, cs in CASES.items():
        if only and name not in only:
            continue
        spec = O.PRESETS[name]
        orc = O.Oracle(spec, max_pos=128, mode=0)
        model = hf_model(spec, orc)
        rng = np.random.default_rng(cs["seed"])
        prompt = rng.integers(0, spec.vocab, size=cs["T"]).astype(np.int32)
        with torch.no_grad():
            ids = torch.from_numpy(prompt.astype(np.int64))[None]
            logits = model(ids).logits[0].float().numpy()
            gen, margins = [], []
            cur = ids
            for _ in range(cs["G"]):
                lg = model(cur).logits[0, -1].float()
                top2 = torch.topk(lg, 2)
                gen.append(int(top2.indices[0])); margins.append(float(top2.values[0] - top2.values[1]))
                cur = torch.cat([cur, top2.indices[:1][None]], dim=1)
        out = os.path.join(ROOT, "tests", "golden", f"hf_{name}.npz")
        np.savez_compressed(out, prompt=prompt, logits=logits.astype(np.float32), gen=np.array(gen, np.int32),
                            margins=np.array(margins, np.float32))
        # immediate self-check so a bad fixture is never written silently
        ol = orc.forward(prompt, all_logits=True)
        print(f"{name}: wrote {out}  max|hf-oracle|={np.abs(ol - logits).max():.3e}  max|logit|={np.abs(logits).max():.3f}")
        orc.close()


if __name__ == "__main__":
    main()
