#!/usr/bin/env python
"""BASELINE config 4 on this engine: DDP synthetic transformer (12 layers, d = 1024, bf16,
seq 1024, batch 8 per rank) with process telemetry sampled at 1 kHz by the native C++ sampler for
``--seconds`` (default 60), then the cross-rank reduce.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 \\
        examples/transformer_1khz_ddp.py --seconds 60 --session-root /tmp/traceml_config4

The traced loop is the stock drop-in (``traceml.init(mode="auto")``, ``with traceml.trace_step(model)``,
``traceml.final_summary()``).  Rank 0 prints one JSON line with what was measured: steps, step
time, process samples committed / drained per rank, achieved sampling rate, late periods, the time
of the final cross-rank reduce, and the diagnosis labels."""
import argparse
import json
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import traceml_b200 as traceml  # noqa: E402


class TinyLM(torch.nn.Module):
    def __init__(self, layers=12, d=1024, heads=16, vocab=32000, seq=1024):
        super().__init__()
        self.emb = torch.nn.Embedding(vocab, d)
        self.pos = torch.nn.Parameter(torch.zeros(seq, d))
        layer = torch.nn.TransformerEncoderLayer(d_model=d, nhead=heads, dim_feedforward=4 * d, dropout=0.0,
                                                 batch_first=True, norm_first=True)
        self.enc = torch.nn.TransformerEncoder(layer, num_layers=layers, enable_nested_tensor=False)
        self.head = torch.nn.Linear(d, vocab, bias=False)

    def forward(self, tokens):
        x = self.emb(tokens) + self.pos[: tokens.shape[1]]
        mask = torch.nn.Transformer.generate_square_subsequent_mask(tokens.shape[1], device=tokens.device)
        return self.head(self.enc(x, mask=mask, is_causal=True))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=60.0)
    ap.add_argument("--hz", type=float, default=1000.0)
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--d-model", type=int, default=1024)
    ap.add_argument("--seq", type=int, default=1024)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--session-root", default=None)
    args = ap.parse_args()

    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    os.environ.setdefault("TRACEML_RING_SLOTS", "131072")  # 60 s at 1 kHz = 60 000 process samples per rank

    traceml.init(mode="auto")
    from traceml_b200 import runtime
    from traceml_b200.runtime import TraceMLRuntime

    torch.manual_seed(1234 + rank)
    vocab = 32000
    model = TinyLM(args.layers, args.d_model, 16, vocab, args.seq).cuda()
    if world > 1:
        model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local])
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
    tokens = [torch.randint(0, vocab, (args.batch, args.seq)).pin_memory() for _ in range(4)]

    drained = {"process": 0, "step_time": 0}

    def sink(kind, rows):
        if kind in drained:
            drained[kind] += len(rows)

    sampler = TraceMLRuntime(interval_sec=0.05, native_process_hz=args.hz, sinks=[sink])
    sampler.start()
    t0 = time.perf_counter()
    steps = 0
    while True:
        tk = tokens[steps % len(tokens)]
        with traceml.trace_step(model):
            tk = tk.to("cuda", non_blocking=True)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                logits = model(tk)
                loss = torch.nn.functional.cross_entropy(logits[:, :-1].reshape(-1, vocab).float(),
                                                         tk[:, 1:].reshape(-1))
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
        steps += 1
        if steps % 8 == 0:  # all ranks stop on the same step
            stop = torch.tensor([1.0 if time.perf_counter() - t0 >= args.seconds else 0.0], device="cuda")
            if world > 1:
                dist.all_reduce(stop, op=dist.ReduceOp.MAX)
            if stop.item() > 0:
                break
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t0
    sampler.stop()
    eng = runtime.get_engine()
    info = {"rank": rank, "steps": steps, "elapsed_s": elapsed, "ms_per_step": elapsed / steps * 1e3,
            "proc_samples_committed": eng.proc_count, "proc_samples_drained": drained["process"],
            "achieved_hz": getattr(sampler, "native_samples", 0) / elapsed,
            "late_periods": getattr(sampler, "native_late", None), "step_rows_drained": drained["step_time"]}
    gathered = [None] * world
    if world > 1:
        dist.all_gather_object(gathered, info)
    else:
        gathered = [info]
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    summary = traceml.final_summary(session_root=args.session_root)
    reduce_ms = (time.perf_counter() - t1) * 1e3
    if rank == 0:
        line = {"config": "BASELINE config 4", "world": world, "layers": args.layers, "d_model": args.d_model,
                "seq": args.seq, "batch_per_rank": args.batch, "dtype": "bf16", "sampler_hz_requested": args.hz,
                "seconds": args.seconds, "ranks": gathered, "final_summary_ms": reduce_ms,
                "step_time": summary["step_time"].get("diagnosis", {}).get("status") if isinstance(summary["step_time"].get("diagnosis"), dict) else None,
                "text_head": summary.get("text", "")[:400]}
        print(json.dumps(line))
        print(summary.get("text", ""))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
