#!/usr/bin/env python
"""Model zoo launcher: download a pre-converted model + tokenizer, write a run script, start `dllama chat`.

    python tools/launch.py <model> [-skip-run] [-skip-script] [-y] [--gpus N]

Same role as the reference's launch.py (launch.py:17-195): model table keyed by name (multi-part files are concatenated),
resumable download with retries, `run_<model>.sh` generation. The run script starts this repo's `dllama` on N local GPUs
instead of building the CPU binary.
"""
from __future__ import annotations

import multiprocessing
import os
import socket
import sys
import time
from urllib.request import Request, urlopen

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def parts(n):
    return [chr(97 + i // 26) + chr(97 + i % 26) for i in range(n)]


HF = "https://huggingface.co/b4rtaz/{repo}/resolve/main/{file}?download=true"


def entry(repo, model_file, tok_file, buffer_type="q80", mode="chat", extra="--max-seq-len 4096", n_parts=0):
    urls = [HF.format(repo=repo, file=f"{model_file}{s}") for s in parts(n_parts)] if n_parts else [HF.format(repo=repo, file=model_file)]
    return dict(model_urls=urls, tokenizer_url=HF.format(repo=repo, file=tok_file), buffer_type=buffer_type, mode=mode, extra=extra)


MODELS = {
    "llama3_1_8b_instruct_q40": entry("Llama-3_1-8B-Q40-Instruct-Distributed-Llama", "dllama_model_llama3.1_instruct_q40.m", "dllama_tokenizer_llama_3_1.t"),
    "llama3_1_405b_instruct_q40": entry("Llama-3_1-405B-Q40-Instruct-Distributed-Llama", "dllama_model_llama31_405b_q40_", "dllama_tokenizer_llama_3_1.t", n_parts=56),
    "llama3_2_1b_instruct_q40": entry("Llama-3_2-1B-Q40-Instruct-Distributed-Llama", "dllama_model_llama3.2-1b-instruct_q40.m", "dllama_tokenizer_llama3_2.t"),
    "llama3_2_3b_instruct_q40": entry("Llama-3_2-3B-Q40-Instruct-Distributed-Llama", "dllama_model_llama3.2-3b-instruct_q40.m", "dllama_tokenizer_llama3_2.t"),
    "llama3_3_70b_instruct_q40": entry("Llama-3_3-70B-Q40-Instruct-Distributed-Llama", "dllama_model_llama-3.3-70b_q40", "dllama_tokenizer_llama-3.3-70b.t", n_parts=11),
    "deepseek_r1_distill_llama_8b_q40": entry("DeepSeek-R1-Distill-Llama-8B-Distributed-Llama", "dllama_model_deepseek-r1-distill-llama-8b_q40.m", "dllama_tokenizer_deepseek-r1-distill-llama-8b.t"),
    "qwen3_0.6b_q40": entry("Qwen3-0.6B-Q40-Distributed-Llama", "dllama_model_qwen3_0.6b_q40.m", "dllama_tokenizer_qwen3_0.6b.t"),
    "qwen3_1.7b_q40": entry("Qwen3-1.7B-Q40-Distributed-Llama", "dllama_model_qwen3_1.7b_q40.m", "dllama_tokenizer_qwen3_1.7b.t"),
    "qwen3_8b_q40": entry("Qwen3-8B-Q40-Distributed-Llama", "dllama_model_qwen3_8b_q40.m", "dllama_tokenizer_qwen3_8b.t"),
    "qwen3_14b_q40": entry("Qwen3-14B-Q40-Distributed-Llama", "dllama_model_qwen3_14b_q40_", "dllama_tokenizer_qwen3_14b.t", n_parts=2),
    "qwen3_30b_a3b_q40": entry("Qwen3-30B-A3B-Q40-Distributed-Llama", "dllama_model_qwen3_30b_a3b_", "dllama_tokenizer_qwen3_30b_a3b.t", n_parts=5),
}


def confirm(message: str) -> bool:
    if "-y" in sys.argv:
        return True
    return input(f'❓ {message} ("Y" if yes): ').upper() in ("Y", "YES")


def download_file(urls, path: str):
    if os.path.isfile(path):
        name = os.path.basename(path)
        if not confirm(f"{name} already exists, do you want to download again?"):
            return
    socket.setdefaulttimeout(30)
    last = time.time()
    with open(path, "wb") as f:
        for url in urls:
            offset, attempts = f.tell(), 8
            start_offset = offset
            print(f"📄 {url}")
            while True:
                try:
                    req = Request(url, headers={"Range": f"bytes={offset - start_offset}-"} if offset > start_offset else {})
                    with urlopen(req) as resp:
                        expected = resp.headers.get("Content-Length")
                        received = 0
                        while True:
                            chunk = resp.read(1 << 16)
                            if not chunk:
                                break
                            f.write(chunk)
                            offset += len(chunk)
                            received += len(chunk)
                            if time.time() - last > 1:
                                sys.stdout.write(f"\rDownloaded {offset // 1024} kB")
                                last = time.time()
                        if expected is not None and received < int(expected):   # connection dropped mid-body: resume, do not truncate
                            raise ConnectionError(f"short read: {received} of {expected} bytes")
                    break
                except Exception as e:   # resume from the bytes already on disk
                    attempts -= 1
                    print(f"\n❌ Error downloading {url}: {e}")
                    if attempts == 0:
                        raise
                    print(f"Retrying download {url}...")
                    time.sleep(1)
    sys.stdout.write(" ✅\n")


def download(name: str, model: dict):
    folder = os.path.join(ROOT, "models", name)
    os.makedirs(folder, exist_ok=True)
    mpath = os.path.join(folder, f"dllama_model_{name}.m")
    tpath = os.path.join(folder, f"dllama_tokenizer_{name}.t")
    download_file(model["model_urls"], mpath)
    download_file([model["tokenizer_url"]], tpath)
    print("📀 All files are downloaded")
    return mpath, tpath


def write_run_file(name: str, command: str) -> str:
    path = os.path.join(ROOT, f"run_{name}.sh")
    with open(path, "w") as f:
        f.write("#!/bin/sh\n\n" + command + "\n")
    os.chmod(path, 0o755)
    return path


def usage():
    print("Usage: python launch.py <model> [-skip-run] [-skip-script] [-y] [--gpus N]\n\nAvailable models:")
    for m in MODELS:
        print(f"  {m}")


def main(argv) -> int:
    if len(argv) < 1 or argv[0] not in MODELS:
        usage()
        return 1
    name = argv[0].replace("-", "_")
    gpus = int(argv[argv.index("--gpus") + 1]) if "--gpus" in argv else 1
    model = MODELS[name]
    mpath, tpath = download(name, model)
    command = (f"{os.path.join(ROOT, 'dllama')} {model['mode']} --model {mpath} --tokenizer {tpath} "
               f"--buffer-float-type {model['buffer_type']} --gpus {gpus} {model['extra']}")
    print("To run Distributed Llama you need to execute:\n--- copy start ---\n\n" + command + "\n\n--- copy end -----")
    if "-skip-script" not in argv:
        print(f"🌻 Created {write_run_file(name, command)} script to easy run")
    if "-skip-run" not in argv and confirm("Do you want to run Distributed Llama?"):
        os.system(command)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
