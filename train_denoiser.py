"""`train_denoiser.py` — the reference's training entry point (train_denoiser.py:1621-1633: `python train_denoiser.py
cfg.yaml` under `accelerate launch` / torchrun) over the libb2f engine.

    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 train_denoiser.py scripts/denoiser/flux_qwen2p5vl_7b_vlm_stage2_512_synthetic.yaml

What runs per step (gpt_image_edit_b200/training.py: Stage2Trainer.step, reference :829-1181): VAE-encode target and
context, flow-matching noising with the resolution-shifted logit-normal sigma, frozen Qwen2.5-VL prefill, MLP2, FLUX
forward with block checkpoints, masked MSE against (noise - x0), backward with per-block recompute, ZeRO-2 gradient
reduce-scatter overlapped with the backward, global-norm clipping, AdamW on the rank's fp32 slice, bf16 all-gather.
One process per GPU over NCCL (RANK / LOCAL_RANK / WORLD_SIZE from the launcher), `seed + rank` data streams.

Replaces accelerate + DeepSpeed (scripts/accelerate_configs/zero2.json) and torch.autograd of the reference.
Out of scope, as SURVEY.md section 2 marks it: the real dataset code (univa/dataset), wandb, EMA, SigLIP/MLP3 branches.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import time
from pathlib import Path

import torch


def build_models(conf, device):
    """(model, vae, pipe, empty_pooled): the frozen stack and the trainable tower (reference :301-478, 795-805)."""
    from gpt_image_edit_b200.text_encoders import encode_prompt
    from univa.serve import cli

    mc = conf.model_config
    model, _, _ = cli.load_main_model_and_processor(mc.pretrained_lvlm_name_or_path, device, mc.synthetic, mc.small,
                                                     task_head=False)        # the training script has no task head
    pipe, tokenizers, text_encoders = cli.load_pipe(model.denoise_tower.denoiser, mc.pretrained_denoiser_name_or_path, device,
                                                    mc.synthetic, mc.small)
    if mc.pretrained_mlp2_path:
        sd = torch.load(mc.pretrained_mlp2_path, map_location="cpu")
        sd = {k.split("denoise_projector.")[-1]: v for k, v in sd.items() if "denoise_projector" in k}
        model.denoise_tower.denoise_projector.load_state_dict(sd)
    _, empty_pooled = encode_prompt(text_encoders, tokenizers, "", 256, device, 1)      # :795-805
    if conf.training_config.drop_t5_rate != 1.0:
        raise SystemExit("drop_t5_rate < 1 needs the T5 prompt embeddings of real captions; the stage yamls use 1.0")
    pipe.text_encoder = pipe.text_encoder_2 = None                                       # :806-808 (frees T5 / CLIP)
    del text_encoders
    torch.cuda.empty_cache()
    return model, pipe.vae, pipe, empty_pooled.to(torch.bfloat16)


def unsupported_settings(conf) -> list:
    """Settings of the reference's schema this engine would otherwise silently ignore: each is named with the reason, and
    main() refuses to start rather than train something else than the yaml says."""
    tc, dc, mc = conf.training_config, conf.dataset_config, conf.model_config
    bad = []
    if tc.mixed_precision != "bf16":
        bad.append(f"training_config.mixed_precision={tc.mixed_precision!r}: the engine computes in bf16 with fp32 master "
                   "weights and gradients (the reference's stage yamls use bf16)")
    if tc.optimizer.lower() != "adamw":
        bad.append(f"training_config.optimizer={tc.optimizer!r}: only AdamW is built")
    if tc.ema_deepspeed_config_file is not None:
        bad.append("training_config.ema_deepspeed_config_file: the EMA engine (univa/utils/create_ema.py) is out of scope; "
                   "the stage-2 yaml leaves it unset")
    if tc.drop_condition_rate:
        bad.append("training_config.drop_condition_rate > 0: prompt dropping happens in the reference's dataset code "
                   "(qwen2vl_dataset.py), which the synthetic triples replace")
    if tc.drop_t5_rate != 1.0:
        bad.append("training_config.drop_t5_rate < 1: needs the T5 embeddings of real captions; the stage yamls use 1.0")
    if dc.dataset_type != "synthetic":
        bad.append(f"dataset_config.dataset_type={dc.dataset_type!r}: only the synthetic triples of BASELINE.json configs[3] "
                   "are available offline (the reference's dataset code is out of scope)")
    if dc.ocr_enhancer:
        bad.append("dataset_config.ocr_enhancer: needs the paddleocr service of univa/utils/get_ocr.py")
    if mc.vlm_residual_image_factor:
        bad.append("model_config.vlm_residual_image_factor > 0 is built for inference only (0.0 in every stage yaml)")
    if not mc.only_tune_image_branch and not mc.only_tune_mlp2 and mc.flux_train_layer_idx is not None:
        bad.append("model_config.only_tune_image_branch=false (FF / text-stream / single-block projection weights) is not built")
    return bad


def resolve_resume_checkpoint(tc, log=print):
    """(directory | None, global step it was written at) for `training_config.resume_from_checkpoint`, by the reference's
    rule (train_denoiser.py:347-374): "latest" picks the `checkpoint-<step>` directory of `output_dir` with the largest
    step; any other value contributes only its BASENAME, looked up under `output_dir` (missing: an error, as
    accelerator.load_state raises there); "latest" with no checkpoint starts a fresh run and says so.  The step is parsed from the directory name.

    One deliberate difference: the reference resets its step counter to 0 after parsing it (:764), so a resumed run counts
    — and names its checkpoints — from 0 again while optimizer and LR schedule continue; here the counter continues from
    the checkpoint's step, which is what `max_train_steps` and the checkpoint names mean."""
    want = tc.resume_from_checkpoint
    if not want:
        return None, 0
    out = Path(tc.output_dir)
    if want != "latest":
        name = os.path.basename(os.path.normpath(str(want)))
    else:
        dirs = sorted((d for d in (os.listdir(out) if out.is_dir() else []) if d.startswith("checkpoint")),
                      key=lambda x: int(x.split("-")[1]))
        name = dirs[-1] if dirs else None
    if name is None:
        log(f"Checkpoint '{want}' does not exist. Starting a new training run.")
        return None, 0
    log(f"Resuming from checkpoint {name}")
    if not (out / name).is_dir():          # the reference fails at this point inside accelerator.load_state
        raise FileNotFoundError(f"resume_from_checkpoint: {out / name} is not a directory")
    return out / name, int(name.split("-")[1])


def prune_checkpoints(output_dir, limit, log=print):
    """Before a new checkpoint is written at most `limit - 1` may remain: the oldest `checkpoint-<step>` directories go
    (train_denoiser.py:1195-1225).  Returns the removed names."""
    if limit is None:
        return []
    out = Path(output_dir)
    old = sorted((d for d in os.listdir(out) if d.startswith("checkpoint")), key=lambda x: int(x.split("-")[1]))
    if len(old) < limit:
        return []
    removing = old[:len(old) - limit + 1]
    log(f"{len(old)} checkpoints already exist, removing {len(removing)} checkpoints")
    log(f"removing checkpoints: {', '.join(removing)}")
    for d in removing:
        shutil.rmtree(out / d)
    return removing


def write_univa_directory(mc, save: Path, trained: dict, proj: dict, log=print):
    """checkpoint-N/univa/: the whole model as a directory `from_pretrained` (and `univa.serve.cli --model_path`) reads, which
    the reference's save hook writes with `save_pretrained` + `processor.save_pretrained` (train_denoiser.py:489-498).  Here
    it is the source checkpoint (`pretrained_lvlm_name_or_path`) re-streamed with the trained tensors replaced — the frozen
    Qwen2.5-VL / FLUX tensors are byte-identical to the source.  A synthetic run has no source directory and writes none
    (its trained tensors are in `denoiser_trainable/` and `denoise_projector.bin`).  -> the directory or None."""
    from gpt_image_edit_b200 import checkpoint as ck

    src = Path(mc.pretrained_lvlm_name_or_path or "")
    if mc.synthetic or not (src.is_dir() and any(src.glob("*.safetensors"))):
        return None
    updates = {"denoise_tower.denoiser." + k: v for k, v in trained.items()}
    updates.update(proj)
    ck.rewrite_checkpoint(src, save / "univa", updates)
    log(f"Saved the model to {save / 'univa'} ({len(updates)} trained tensors over {src})")
    return save / "univa"


def load_checkpoint(path: Path, trainer, rank: int, device):
    """accelerator.load_state (:769) for this engine: the rank's optimizer partition — which also restores the bf16
    weights the model computes with (ShardedAdamW.load_state_dict) — and the rank's random streams."""
    trainer.opt.load_state_dict(torch.load(path / f"optimizer_rank{rank}.pt", map_location=device))
    rs = path / f"random_states_{rank}.pkl"
    if rs.exists():
        st = torch.load(rs, map_location="cpu", weights_only=False)
        torch.set_rng_state(st["torch"])
        if st.get("noise") is not None and getattr(trainer, "gen", None) is not None:
            trainer.gen.set_state(st["noise"])


def save_checkpoint(conf, trainer, model, step: int, rank: int, world: int):
    """checkpoint-{step}/: the trainable tensors under their diffusers names (safetensors, rank 0), denoise_projector.bin
    (reference :1231-1236), this rank's optimizer partition and random streams (ZeRO: one file per rank, :1229
    accelerator.save_state writes `random_states_<rank>.pkl` the same way)."""
    from gpt_image_edit_b200 import checkpoint as ck

    tc = conf.training_config
    out = Path(tc.output_dir)
    out.mkdir(parents=True, exist_ok=True)
    if rank == 0:
        prune_checkpoints(out, tc.checkpoints_total_limit)
    save = out / f"checkpoint-{step}"
    save.mkdir(parents=True, exist_ok=True)
    if rank == 0:
        den = model.denoise_tower.denoiser.state_dict()
        from gpt_image_edit_b200.training import check_param_is_in_components, get_trainable_params, trained_flux_layers
        comps = get_trainable_params(trained_flux_layers(conf.model_config), model.denoise_tower.denoiser.config.num_layers,
                                     conf.model_config.only_tune_image_branch)
        trained = {k: v for k, v in den.items() if check_param_is_in_components("denoise_tower.denoiser." + k, comps)}
        ck.save_state_dict(trained, save / "denoiser_trainable")
        proj = {}
        if conf.model_config.only_tune_mlp2 or conf.model_config.with_tune_mlp2:
            proj = {f"denoise_tower.denoise_projector.{k}": v.cpu() for k, v in
                    model.denoise_tower.denoise_projector.state_dict().items()}
            torch.save(proj, save / "denoise_projector.bin")
        write_univa_directory(conf.model_config, save, trained, proj)
        (save / "trainer_state.json").write_text(json.dumps({"global_step": step, "world_size": world}))
    torch.save(trainer.opt.state_dict(), save / f"optimizer_rank{rank}.pt")
    gen = getattr(trainer, "gen", None)
    torch.save({"torch": torch.get_rng_state(), "noise": None if gen is None else gen.get_state().cpu()},
               save / f"random_states_{rank}.pkl")
    return save


def main(conf):
    from gpt_image_edit_b200 import distributed as D
    from gpt_image_edit_b200.training import Stage2Trainer
    from univa.training.synthetic_data import SyntheticEditDataset, collate

    if not torch.cuda.is_available():
        raise SystemExit("train_denoiser.py runs on H100s through libb2f; there is no CPU path")
    tc, dc, mc = conf.training_config, conf.dataset_config, conf.model_config
    world, rank, local_rank = D.env_world()
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    D.init_from_env(device=device)
    torch.manual_seed(tc.seed + rank)                                  # set_seed(seed, device_specific=True) (:290)
    bad = unsupported_settings(conf)
    if bad:
        raise SystemExit("train_denoiser.py cannot honour this configuration:\n  - " + "\n  - ".join(bad))
    if tc.profile_out_dir is not None and rank == 0:
        print("profile_out_dir is ignored: use libb2f's CUDA-event profiler (bench.py --workload train512) or ncu "
              "(scripts/profile_train.py)", flush=True)
    model, vae, pipe, empty_pooled = build_models(conf, device)
    if world > 1:      # every rank starts from rank 0's weights (DeepSpeed broadcasts parameters at initialize())
        D.broadcast_weights(list(model.denoise_tower.denoiser._store.values()) +
                            list(model.denoise_tower.denoise_projector.state_dict().values()))
    trainer = Stage2Trainer(model, vae, pipe, tc, mc, empty_pooled)
    trainer.gen = torch.Generator(device=device).manual_seed(tc.seed + rank)
    n_train = sum(p.storage.numel() for p in trainer.params)
    if rank == 0:
        print(f"trainable tensors: {len(trainer.params)}  parameters: {n_train / 1e9:.3f} B  world: {world}  "
              f"ZeRO-2 buckets: {sum(b is not None for b in trainer.opt.buckets)}", flush=True)
    ck, start = resolve_resume_checkpoint(tc, log=print if rank == 0 else (lambda *a: None))
    if ck is not None:
        load_checkpoint(ck, trainer, rank, device)
        trainer.global_step = start
    data = SyntheticEditDataset(dc.height, dc.width, dc.synthetic_len, seed=tc.seed + rank, target_sizes=dc.synthetic_target_sizes)
    loader = torch.utils.data.DataLoader(data, batch_size=dc.batch_size, collate_fn=collate, num_workers=0,
                                         pin_memory=dc.pin_memory)
    max_steps = tc.max_train_steps or (len(loader) * tc.num_train_epochs // tc.gradient_accumulation_steps)
    t0 = time.time()
    for batch in loader:
        out = trainer.step(batch)
        if not out["stepped"]:
            continue
        step = trainer.global_step
        loss = out["loss"].detach().clone()
        if world > 1:                                                   # accelerator.gather(loss) (:1168)
            torch.distributed.all_reduce(loss)
            loss /= world
        if rank == 0:
            dt = time.time() - t0
            print(f"step {step}  loss {loss.item():.5f}  grad_norm {out['grad_norm'].item():.4f}  lr {out['lr']:.3e}  "
                  f"{dc.batch_size * tc.gradient_accumulation_steps * world * (step - start) / max(dt, 1e-9):.3f} samples/s",
                  flush=True)
        if step % tc.checkpointing_steps == 0:
            path = save_checkpoint(conf, trainer, model, step, rank, world)
            if rank == 0:
                print(f"Saved state to {path}", flush=True)
        if step >= max_steps:
            break
    D.barrier()
    return trainer


if __name__ == "__main__":
    from univa.training.configuration_denoise import load_config

    parser = argparse.ArgumentParser()
    parser.add_argument("config", type=str)
    main(load_config(parser.parse_args().config))
