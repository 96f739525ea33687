#!/bin/bash
# Start root + workers on N local GPUs in one command (the analogue of the reference's examples/n-workers.sh, which
# spawns N TCP workers in `screen`): here every rank is a torchrun-managed process bound to one GPU.
#
#   N=8 MODEL=model.m TOKENIZER=tok.t bash examples/n-gpus.sh inference --prompt "Hello" --steps 64
#   NATIVE=1 N=8 ... bash examples/n-gpus.sh inference ...     # the C++ binary: the root forks one worker per GPU, no Python
cd "$(dirname "$0")/.."
N=${N:-2}
if [ -z "$MODEL" ] || [ -z "$TOKENIZER" ]; then
  echo "Usage: N=<gpus> MODEL=<path.m> TOKENIZER=<path.t> $0 {inference|chat|perplexity} [dllama flags]"
  exit 1
fi
MODE=${1:-chat}; shift
if [ -n "$NATIVE" ]; then
  exec ./dllama-native "$MODE" --model "$MODEL" --tokenizer "$TOKENIZER" --gpus "$N" "$@"
fi
exec python -m torch.distributed.run --nnodes=1 --nproc-per-node="$N" --master-addr 127.0.0.1 --master-port "${PORT:-29500}" \
  -m distributed_llama_b200.apps.cli "$MODE" --model "$MODEL" --tokenizer "$TOKENIZER" --buffer-float-type q80 "$@"
