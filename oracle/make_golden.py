"""Regenerates tests/golden/reference_perplexity.json: the reference binary's `dllama perplexity` output (per-token probabilities and
the perplexity line) on the synthetic tiny models of tests/conftest.py. Needs oracle/_ref/dllama (oracle/build_reference.sh).

    python oracle/make_golden.py
"""
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PROMPT = "Hello world, the model is a llama and the token"
MODELS = ("tiny-llama", "tiny-llama31", "tiny-qwen3", "tiny-qwen3-moe")


def main():
    from distributed_llama_b200.models.config import get_config
    from distributed_llama_b200.models.synthetic import write_synthetic_model, write_synthetic_tokenizer

    exe = os.path.join(ROOT, "oracle", "_ref", "dllama")
    out = {"prompt": PROMPT, "command": "dllama perplexity --buffer-float-type q80 --nthreads 2", "models": {}}
    with tempfile.TemporaryDirectory() as d:
        for name in MODELS:
            cfg = get_config(name)
            m, t = os.path.join(d, name + ".m"), os.path.join(d, name + ".t")
            write_synthetic_model(m, cfg, seed=7)     # same files as the tmp_models fixture
            write_synthetic_tokenizer(t, cfg.vocab_size, style="chatml" if "qwen" in name else "llama3")
            r = subprocess.run([exe, "perplexity", "--model", m, "--tokenizer", t, "--buffer-float-type", "q80", "--prompt", PROMPT,
                                "--nthreads", "2"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300, check=True)
            probs = [float(x) for x in re.findall(r"prob=([0-9.eE+-]+)", r.stdout)]
            ppl = float(re.search(r"perplexity: ([0-9.]+)", r.stdout).group(1))
            out["models"][name] = {"probs": probs, "perplexity": ppl}
    path = os.path.join(ROOT, "tests", "golden", "reference_perplexity.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print(path)


if __name__ == "__main__":
    main()
