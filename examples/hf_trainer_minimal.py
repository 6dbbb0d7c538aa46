#!/usr/bin/env python
"""BASELINE config 5 on this engine: the reference's ``examples/huggingface_trainer_minimal.py``
(TinyMLP, 200 steps, synthetic data) through the KEPT, UNMODIFIED ``TraceMLTrainer`` of the
reference package (``oracle/_ref/traceml/integrations/huggingface.py:22-83``: a
``transformers.Trainer`` subclass whose ``training_step`` runs inside the reference's own
``trace_step``), bound to this engine by ``traceml_b200.shim`` (INTEGRATION.md option B), bf16, one
rank per GPU.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 \\
        examples/hf_trainer_minimal.py --session-root /tmp/traceml_config5

``transformers.Trainer`` needs the ``accelerate`` package (transformers >= 4.x raises ImportError in
``Trainer.__init__`` without it) and this image has none.  The script first tries the real
``Trainer``; if that fails it says exactly why and falls back to a stand-in base class that
reproduces the part of the Trainer loop the integration touches -- ``training_step(model, inputs)``
= forward (``model(**inputs)["loss"]``) + backward under bf16 autocast on the DDP-wrapped model,
optimizer step and zero_grad outside it, ``max_steps`` -- so that the kept subclass, unmodified,
drives the engine exactly as it would under Hugging Face.  Rank 0 prints one JSON line and writes
``final_summary.{json,txt}``.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.utils.data import DataLoader, Dataset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))   # the installed reference package
os.environ.setdefault("TRACEML_LOGS_DIR", "/tmp/traceml_ref_logs")
import traceml  # noqa: E402  -- the REFERENCE's package: its API, patches and integrations, unmodified
import traceml_b200  # noqa: E402
from traceml_b200 import shim  # noqa: E402

SEED, INPUT_DIM, HIDDEN_DIM, NUM_CLASSES, NUM_SAMPLES, BATCH_SIZE, MAX_STEPS = 42, 128, 256, 10, 4096, 64, 200


class SyntheticClassificationDataset(Dataset):
    def __init__(self, num_samples):
        self.x = torch.randn(num_samples, INPUT_DIM)
        self.y = torch.randint(0, NUM_CLASSES, (num_samples,))

    def __len__(self):
        return len(self.y)

    def __getitem__(self, idx):
        return {"inputs": self.x[idx], "labels": self.y[idx]}


class TinyMLPForTrainer(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(INPUT_DIM, HIDDEN_DIM), nn.ReLU(), nn.Linear(HIDDEN_DIM, NUM_CLASSES))
        self.loss_fn = nn.CrossEntropyLoss()

    def forward(self, inputs=None, labels=None):
        logits = self.net(inputs)
        return {"loss": self.loss_fn(logits, labels) if labels is not None else None, "logits": logits}


class StandInTrainer:
    """The slice of ``transformers.Trainer`` the integration relies on."""

    def __init__(self, model=None, args=None, train_dataset=None, **_):
        self.model, self.args, self.train_dataset = model, args, train_dataset

    def training_step(self, model, inputs, *a, **k):
        model.train()
        inputs = {k_: v.to("cuda", non_blocking=True) for k_, v in inputs.items()}
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=self.args["bf16"]):
            loss = model(**inputs)["loss"]
        loss.backward()
        return loss.detach()

    def train(self):
        local, world = int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
        model = self.model.cuda()
        if world > 1:
            model = nn.parallel.DistributedDataParallel(model, device_ids=[local])
        opt = torch.optim.AdamW(model.parameters(), lr=5e-5)
        sampler = torch.utils.data.distributed.DistributedSampler(self.train_dataset) if world > 1 else None
        loader = DataLoader(self.train_dataset, batch_size=self.args["per_device_train_batch_size"], sampler=sampler,
                            shuffle=sampler is None, pin_memory=True)
        step = 0
        while step < self.args["max_steps"]:
            for inputs in loader:
                self.training_step(model, inputs)
                opt.step()
                opt.zero_grad(set_to_none=True)
                step += 1
                if step >= self.args["max_steps"]:
                    break
        return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--session-root", default=None)
    ap.add_argument("--max-steps", type=int, default=MAX_STEPS)
    args = ap.parse_args()
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    torch.manual_seed(SEED)
    shim.install()              # the reference's seam now records through libtraceml_b200.so
    traceml.init(mode="auto")   # the reference's own init

    why, used = None, "transformers.Trainer"
    trainer = None
    try:
        from transformers import TrainingArguments

        from traceml.integrations.huggingface import TraceMLTrainer

        targs = TrainingArguments(output_dir="/tmp/hf_minimal_output", per_device_train_batch_size=BATCH_SIZE,
                                  max_steps=args.max_steps, logging_steps=50, save_strategy="no", report_to="none",
                                  disable_tqdm=True, remove_unused_columns=False, bf16=True)
        trainer = TraceMLTrainer(model=TinyMLPForTrainer(), args=targs,
                                 train_dataset=SyntheticClassificationDataset(NUM_SAMPLES), traceml_enabled=True)
    except Exception as exc:  # noqa: BLE001 -- recorded, then the stand-in base class takes over
        why = f"{type(exc).__name__}: {exc}"[:400]
        import transformers

        for mod in [m for m in sys.modules if m.startswith("traceml.integrations.huggingface")]:
            del sys.modules[mod]
        transformers.Trainer = StandInTrainer  # the kept subclass is defined over whatever `Trainer` is
        from traceml.integrations.huggingface import TraceMLTrainer

        used = "stand-in Trainer base (transformers.Trainer unusable here)"
        trainer = TraceMLTrainer(model=TinyMLPForTrainer(),
                                 args={"per_device_train_batch_size": BATCH_SIZE, "max_steps": args.max_steps, "bf16": True},
                                 train_dataset=SyntheticClassificationDataset(NUM_SAMPLES), traceml_enabled=True)
    trainer.train()
    torch.cuda.synchronize()
    summary = traceml_b200.final_summary(session_root=args.session_root)
    if rank == 0:
        st = summary["step_time"]
        print(json.dumps({"config": "BASELINE config 5", "world": world, "trainer_base": used,
                          "real_trainer_error": why, "max_steps": args.max_steps, "dtype": "bf16",
                          "top_level_keys": sorted(summary.keys()),
                          "step_time_keys": sorted(st.keys()) if isinstance(st, dict) else None,
                          "training_steps": (st.get("metadata") or {}).get("training_total_steps") if isinstance(st, dict) else None}))
        print(summary.get("text", ""))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
