"""Native tuning worker — the process behind the controller's `python /tuning/train.py ...` (cmd/tuning/train.py).

Flow (reference line in brackets):
  parse argv [parser.get_train_args, train.py:313]  ->  block_size -> cutoff_len [323-325]  ->  tokenizer [337]
  -> CSV + column rename [339-340] -> llama2 template + label masking [342, 58-135]
  -> one rank per GPU (the reference: one Ray actor per worker, train.py:353-368) -> data-parallel LoRA-SFT steps on
     libdtxtune (replaces trainer_init_per_worker + HF Trainer.train(), train.py:138-299)
  -> log every 10 optimizer steps [198; callback.py:95-155] -> eval_loss / eval_perplexity every 10 steps when
     --evaluation_path is set [186-190; trainer.py:324-327]
  -> PEFT adapter dir under storage_path [300-305] -> /home/ray/checkpoint_path without trailing newline [379-389]
Exit status: 0 on success, non-zero on any error (the controller maps it to RayJob SUCCEEDED/FAILED).

Multi-GPU: rank 0 creates the NCCL unique id and re-executes itself once per extra GPU with DTX_RANK/DTX_NCCL_ID in the
environment (single node, one process per GPU, no torch.distributed needed); a watchdog thread takes the job down
when a child rank dies, and a failure on rank 0 kills the children.
"""
from __future__ import annotations

import math
import os
import subprocess
import sys
import threading
import time
from typing import List, Optional

import numpy as np

from .. import lib as L
from . import data as D
from . import model_io
from .callback import LogCallback
from .parser import TrainArgs, get_train_args

CHECKPOINT_PATH_FILE = os.environ.get("DTX_CHECKPOINT_PATH_FILE", "/home/ray/checkpoint_path")


def total_optimizer_steps(n_examples: int, world: int, batch: int, grad_accum: int, epochs: float, max_steps: int) -> int:
    """HF Trainer: len(dataloader) = ceil(shard / batch) (the last partial batch is kept), num_update_steps_per_epoch =
    max(len(dataloader) // grad_accum, 1), max_steps = ceil(epochs * that)."""
    per_epoch = max(D.steps_per_epoch(n_examples, world, batch) // max(1, grad_accum), 1)
    return max_steps if max_steps > 0 else int(math.ceil(epochs * per_epoch))


def evaluate(tr, eval_set, rank: int, world: int, B: int, seq_len: int, pad_id: int, eval_batch: int, seed: int) -> Optional[float]:
    """SFTTrainer.evaluate's eval_loss (cmd/tuning/trainer.py:324-327): HF runs the eval split in batches of
    per_device_eval_batch_size on every process, repeats each batch's token-mean loss once per sample, gathers and averages.
    The native step has one static micro-batch, so rows come back with (sum of token losses, valid tokens) and the host
    forms HF's batches of `eval_batch` consecutive samples from them."""
    sums, cnts = [], []
    for ids, lab, lens in D.epoch_batches(eval_set, rank, world, B, seq_len, pad_id, 0, seed, varlen=True, shuffle=False):
        s_, c_ = tr.eval_rows(ids, lab, lens)
        real = int((lens > 0).sum())
        sums += s_[:real].tolist()
        cnts += c_[:real].tolist()
    tot, n = 0.0, 0
    for i in range(0, len(sums), eval_batch):
        c = sum(cnts[i:i + eval_batch])
        k = len(sums[i:i + eval_batch])
        tot += k * (sum(sums[i:i + eval_batch]) / max(c, 1))
        n += k
    red = tr.allreduce_host([tot, float(n)])
    return float(red[0] / red[1]) if red[1] > 0 else None


def run_rank(a: TrainArgs, rank: int, world: int, nccl_id: Optional[bytes], tokenizer=None) -> Optional[str]:
    if a.quantization and a.quantization not in ("int4", "int8"):
        raise L.DtxError(-1, f"--quantization {a.quantization}: expected int4 or int8 (cmd/tuning/train.py:224-234)")
    if a.fp16 and rank == 0:
        # finetune_controller.go:506 plumbs --fp16 (HF AMP + DeepSpeed dynamic loss scaling, ds_config.json:6-8).  The native step
        # computes in bf16 with fp32 accumulation: same 16-bit storage, wider exponent, so no loss scaling and no skipped steps.
        print("[dtx] --fp16 true: the native worker computes in bf16 (fp32 accumulate); fp16 loss scaling does not apply", flush=True)
    if tokenizer is None:
        from transformers import AutoTokenizer  # host-side tokenisation only
        tokenizer = AutoTokenizer.from_pretrained(a.model_name_or_path)
    D.fix_tokenizer(tokenizer)
    cutoff_len = a.block_size if a.block_size > 0 else 1024  # train.py:51,323-325
    rows = D.read_csv_rows(a.train_path, a.columns_map())
    dataset = D.build_dataset(rows, tokenizer, cutoff_len)
    if not dataset:
        raise RuntimeError("Empty dataset!")  # train.py:133
    if len(dataset) < world:
        raise RuntimeError(f"{len(dataset)} training examples cannot be split over {world} workers")
    eval_set = dataset if a.evaluation_path else None  # the reference re-reads the TRAIN file for eval (train.py:347)

    # The reference parses --finetuning_type and then wraps LoRA regardless (cmd/tuning/train.py:266-280): a drop-in must do the
    # same.  Full-parameter SFT (BASELINE.json configs[3]) is an explicit opt-in on top: DTX_HONOR_FINETUNING_TYPE=1.
    full = a.finetuning_type == "full" and os.environ.get("DTX_HONOR_FINETUNING_TYPE") == "1"
    mc = model_io.load_model_config(a.model_name_or_path, full_finetune=full)
    seq_len = D.static_seq_len(cutoff_len)
    model_io.check_attention_window(a.model_name_or_path, seq_len)
    B, GA = a.per_device_train_batch_size, max(1, a.gradient_accumulation_steps)
    total = total_optimizer_steps(len(dataset), world, B, GA, a.num_train_epochs, a.max_steps)
    if a.finetuning_type != "lora" and not full and rank == 0:
        print(f"[dtx] --finetuning_type {a.finetuning_type} is ignored like in the reference worker (LoRA is always applied); "
              "set DTX_HONOR_FINETUNING_TYPE=1 for native full-parameter SFT", flush=True)
    tc = L.TrainConfig(micro_batch=B, seq_len=seq_len, total_steps=total, lora_r=a.lora_rank, lora_alpha=a.lora_alpha,
                       lora_dropout=a.lora_dropout, lora_target=tuple(a.lora_target), lr=a.learning_rate, weight_decay=a.weight_decay,
                       beta1=a.adam_beta1, beta2=a.adam_beta2, eps=a.adam_epsilon, max_grad_norm=a.max_grad_norm,
                       sched=a.lr_scheduler_type, warmup_steps=a.warmup_steps, grad_accum=GA, seed=a.seed, full_finetune=full)
    for kv in filter(None, os.environ.get("DTX_OPTIONS", "").split(",")):  # library A/B switches, e.g. DTX_OPTIONS=varlen_pack=0
        name, sep, value = kv.partition("=")
        if not sep or not value.strip().lstrip("-").isdigit():
            raise L.DtxError(-1, f"DTX_OPTIONS entry {kv!r}: expected name=integer")
        L.set_option(name.strip(), int(value))  # an unknown name raises (DTX_ERR_INVALID)
    device = int(os.environ.get("DTX_DEVICE", rank))
    tr = L.Trainer(mc, tc, device=device, rank=rank, world=world, nccl_id=nccl_id)
    if rank == 0:  # --gradient_checkpointing is ignored (the reference hard-codes it): the library picks what fits the device
        keep, layer = (L.plan_device_bytes(mc, tc, world, k) for k in ("keep", "layer"))
        print(f"[dtx] activations: {'recompute per layer' if tr.recompute == 'layer' else 'keep all'} "
              f"(planned device bytes per rank: keep all {keep / 1e9:.1f} GB, recompute per layer {layer / 1e9:.1f} GB)", flush=True)
    if os.environ.get("DTX_RANDOM_INIT"):  # benchmarking / scheduling harnesses: config.json only, N(0, 0.02) weights on the device
        tr.init_random_weights(int(os.environ["DTX_RANDOM_INIT"]))
    else:
        model_io.load_weights_into(tr, a.model_name_or_path)
    if a.quantization:  # QLoRA: packed NF4 base (train.py:224-230); int8 is refused by the library
        tr.quantize_base(a.quantization)
    if not full:
        tr.init_lora(a.seed)
    cb = LogCallback(a.output_dir, total, a.metrics_export_address, a.uid) if rank == 0 else None

    pad_id = tokenizer.pad_token_id
    steps_in_epoch = D.steps_per_epoch(len(dataset), world, B)  # len(dataloader)
    step, window, micro_losses, t0 = 0, [], [], time.time()
    batched, tokens = 0, 0  # HF total_batched_samples: accumulation runs across epoch boundaries
    t_first, tok_first, t_last = None, 0, None  # steady state: from the end of the first optimizer step to the end of the last
    groups_sum = 0  # length groups the ragged micro-batches were run as (DESIGN.md 2.2)
    epoch = 0
    while step < total:
        for i, (ids, labels, lens) in enumerate(D.epoch_batches(dataset, rank, world, B, seq_len, pad_id, epoch, a.seed, varlen=True)):
            batched += 1
            # HF 4.34 Trainer._inner_training_loop: step when total_batched_samples % GA == 0, or at the end of an epoch that
            # holds no more than GA batches
            last_of_short_epoch = steps_in_epoch <= GA and (i + 1) == steps_in_epoch
            boundary = batched % GA == 0 or last_of_short_epoch
            loss, gnorm, lr, stepped = tr.step(ids, labels, lens, force_step=boundary)
            tokens += int(lens.sum())
            groups_sum += tr.last_step_groups
            micro_losses.append(loss)
            if not stepped:
                continue
            step += 1
            t_last = time.time()
            if t_first is None:
                t_first, tok_first = t_last, tokens
            window.append(float(np.sum(micro_losses)) / GA)  # HF divides every micro-batch loss by GA
            micro_losses = []
            frac_epoch = epoch + (i + 1) / steps_in_epoch
            if cb:
                cb.on_step_end(step)
            if step % a.logging_steps == 0:
                if cb:  # HF logs the mean loss since the last log and the *next* lr
                    cb.on_log(float(np.mean(window)), a.learning_rate * L.lr_lambda(a.lr_scheduler_type, step, a.warmup_steps, total),
                              frac_epoch)
                window = []
                if eval_set is not None:  # evaluation_strategy="steps" with eval_steps = logging_steps = 10 (train.py:186-198)
                    ev = evaluate(tr, eval_set, rank, world, B, seq_len, pad_id, a.per_device_eval_batch_size, a.seed)
                    if cb and ev is not None:
                        cb.on_eval(ev, math.exp(ev), frac_epoch)  # eval_perplexity = exp(eval_loss), trainer.py:324-327
            if step >= total:
                break
        epoch += 1
    ckpt = None
    if rank == 0:
        name = f"TorchTrainer_{time.strftime('%Y-%m-%d_%H-%M-%S')}/checkpoint_000000"
        ckpt = os.path.join(a.storage_path, name)
        if full:  # trainer.save_model of a full fine-tune writes the whole model
            weights = tr.export_weights()
            for out in (ckpt, a.output_dir):
                model_io.save_full_model(out, weights, a.model_name_or_path)
        else:
            adapter = tr.export_adapter()
            for out in (ckpt, a.output_dir):
                model_io.save_peft_adapter(out, adapter, base_model=a.model_name_or_path, r=a.lora_rank, alpha=a.lora_alpha,
                                           dropout=a.lora_dropout, target_modules=a.lora_target)
        dt = time.time() - t0
        print(f"train_runtime {dt:.1f}s, {step} optimizer steps, {tokens} real tokens on rank 0 ({tokens / max(dt, 1e-9):.1f} tokens/s/rank)",
              flush=True)
        if step > 1 and t_last > t_first:  # without the first step (lazy CUDA / NCCL initialisation) and the checkpoint writes
            print(f"steady_state {t_last - t_first:.3f}s, {step - 1} optimizer steps, {tokens - tok_first} real tokens on rank 0 "
                  f"({(tokens - tok_first) / (t_last - t_first):.1f} tokens/s/rank), {groups_sum / max(batched, 1):.2f} length groups per micro-batch",
                  flush=True)
    tr.close()
    return ckpt


def _watch_children(children, stop) -> None:
    """A rank that dies (OOM, bad device) leaves its peers blocked inside ncclAllReduce forever: poll the children and take
    the whole job down with a non-zero status as soon as one exits early."""
    while not stop.is_set():
        for c in children:
            rc = c.poll()
            if rc is not None and rc != 0:
                print(f"[dtx] worker rank process {c.pid} exited with status {rc}: aborting the job", file=sys.stderr, flush=True)
                for o in children:
                    if o.poll() is None:
                        o.kill()
                os._exit(rc if rc > 0 else 1)
        stop.wait(0.5)


def main(argv: Optional[List[str]] = None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    a = get_train_args(argv)
    rank = int(os.environ.get("DTX_RANK", "0"))
    world = max(1, a.num_workers)
    nccl_id = bytes.fromhex(os.environ["DTX_NCCL_ID"]) if "DTX_NCCL_ID" in os.environ else None
    children, stop = [], threading.Event()
    if world > 1 and rank == 0 and nccl_id is None:
        nccl_id = L.nccl_unique_id()
        for r in range(1, world):
            env = dict(os.environ, DTX_RANK=str(r), DTX_NCCL_ID=nccl_id.hex())
            children.append(subprocess.Popen([sys.executable, "-m", "datatunerx_b200.tuning.train"] + argv, env=env))
        threading.Thread(target=_watch_children, args=(children, stop), daemon=True).start()
    try:
        ckpt = run_rank(a, rank, world, nccl_id)
    except BaseException:
        stop.set()
        for c in children:  # never leave orphans spinning in NCCL
            if c.poll() is None:
                c.kill()
        raise
    rc = 0
    for c in children:
        rc = rc or c.wait()
    stop.set()
    if rc:
        return rc
    if rank == 0 and ckpt:
        print(f"result path {ckpt}")
        d = os.path.dirname(CHECKPOINT_PATH_FILE)
        if d and not os.path.exists(d):
            os.makedirs(d)
        with open(CHECKPOINT_PATH_FILE, "w", encoding="utf-8") as f:
            f.write(ckpt)  # no trailing newline: the controller `cat`s it verbatim (finetune_controller.go:201-212)
    return 0


if __name__ == "__main__":
    sys.exit(main())
