"""GEdit sampling driver over the libb2f engine — the multi-GPU caller of the hot path
(reference univa/eval/gedit/step1_gen_samples.py:33-36, 82-92, 95-214, 225-250; SURVEY.md §8e).

    torchrun --nproc-per-node N -m univa.eval.gedit.step1_gen_samples cfg.yaml [--output_dir ...]

Same contract as the reference: a prompt file {key: {"prompt": ..., "id": <relative image path>}}, one full
model replica per rank (no collective during sampling), items strided `rank::world_size`, `seed + rank` seeding of the
default generators (the pipeline is given no generator of its own),
outputs written to `output_dir/<id>` and skipped when they already exist, generation size from
`pick_ratio(any_17ratio)` + `compute_size(stride 16, anchor height*width)`, a fixed 448x448 view for the VLM,
an empty T5 prompt unless `joint_with_t5`.  Judges / metrics (step2) are out of scope.
"""
from __future__ import annotations

import argparse
import json
import os
from pathlib import Path

import numpy as np
import torch
import yaml

from gpt_image_edit_b200 import distributed as D
from gpt_image_edit_b200.image_io import image_to_condition_tensor, qwen_pixel_values, resize_u8
from gpt_image_edit_b200.text_encoders import encode_prompt
from univa.eval.configuration_eval import EvalConfig
from univa.serve import cli
from univa.utils.anyres_util import compute_size, pick_ratio


def load_items(prompt_path, output_dir) -> list:
    """[(prompt, output_path, key, relative image path)] in file order (:228-237)."""
    with open(prompt_path) as f:
        data = json.load(f)
    return [(v["prompt"], os.path.join(output_dir, v["id"]), k, v["id"]) for k, v in data.items()]


def generation_size(orig_h: int, orig_w: int, height: int, width: int):
    """(gen_h, gen_w): nearest of the 17 aspect ratios, then the anchor area on a stride-16 grid (:100-114)."""
    rw, rh = pick_ratio(orig_h, orig_w, anyres="any_17ratio")
    return compute_size(rw, rh, stride=16, anchor_pixels=height * width)


@torch.no_grad()
def run_model_and_return_samples(args: EvalConfig, state: dict, prompt_text: str, image1, image2=None):
    from PIL import Image

    if image2 is not None:
        raise NotImplementedError("one context image per edit (the reference pipeline consumes image[0] only)")
    img = np.asarray(Image.open(image1).convert("RGB"))
    gen_h, gen_w = generation_size(img.shape[0], img.shape[1], args.height, args.width)
    dev = state["device"]
    if state.get("processor") is not None:
        # the reference's prompt path (:119-151): a fixed 448x448 view for the VLM, chat template, system turn dropped
        content = [{"type": "image", "image": image1, "resized_height": 448, "resized_width": 448}]
        if prompt_text:
            content.append({"type": "text", "text": prompt_text})
        inputs = cli.prepare_inputs(state["processor"], [{"role": "user", "content": content}], dev)
        lvlm = state["model"](inputs.input_ids, pixel_values=inputs["pixel_values"], attention_mask=inputs.attention_mask,
                              image_grid_thw=inputs["image_grid_thw"], output_type="denoise_embeds")
    else:       # --synthetic only: no tokenizer files offline (cli.load_main_model_and_processor raises otherwise)
        pix, grid = qwen_pixel_values(resize_u8(img, 448, 448))
        input_ids = cli.synthetic_chat_tokens(pix.shape[0] // 4).to(dev)
        lvlm = state["model"](input_ids, pixel_values=pix.to(dev), attention_mask=torch.ones_like(input_ids),
                              image_grid_thw=grid, output_type="denoise_embeds")
    t5, pooled = encode_prompt(state["text_encoders"], state["tokenizers"], prompt_text if args.joint_with_t5 else "", 256, dev, 1)
    embeds = t5 if args.only_use_t5 else (torch.cat([lvlm, t5], dim=1) if args.joint_with_t5 else lvlm)
    # no `generator=`, as in the reference (:195-204): the noise comes from the device's default generator, which main()
    # seeded with seed + rank, so the i-th image of a rank continues that stream exactly as it does there
    return state["pipe"](image=image_to_condition_tensor(img).to(dev), prompt_embeds=embeds, pooled_prompt_embeds=pooled,
                         height=gen_h, width=gen_w, num_inference_steps=args.num_inference_steps,
                         guidance_scale=args.guidance_scale, num_images_per_prompt=args.num_images_per_prompt).images


def main(args: EvalConfig):
    if not torch.cuda.is_available():
        raise SystemExit("the sampling driver runs on H100s through libb2f; there is no CPU path")
    world, rank, local_rank = D.env_world()
    device = torch.device("cuda", local_rank)
    torch.cuda.set_device(device)
    D.init_from_env(device=device)
    args.local_rank, args.world_size = rank, world
    import random
    random.seed(D.rank_seed(args.seed, rank))                                 # set_seed(seed, rank, device_specific=True) (:33-43)
    np.random.seed(D.rank_seed(args.seed, rank))
    torch.manual_seed(D.rank_seed(args.seed, rank))                           # CPU and every CUDA device
    model, _, processor = cli.load_main_model_and_processor(args.pretrained_lvlm_name_or_path, device, args.synthetic, args.small,
                                                            min_pixels=args.min_pixels, max_pixels=args.max_pixels, task_head=False)   # :45-56
    pipe, tokenizers, text_encoders = cli.load_pipe(model.denoise_tower.denoiser, args.pretrained_denoiser_name_or_path, device,
                                                    args.synthetic, args.small)
    state = dict(model=model, pipe=pipe, tokenizers=tokenizers, text_encoders=text_encoders, device=device, processor=processor)
    os.makedirs(args.output_dir, exist_ok=True)
    todo = D.shard(load_items(args.gedit_prompt_path, args.output_dir), rank, world)     # inference_list[rank::world] (:239)
    done = 0
    for prompt, out_path, _key, rel in todo:
        if os.path.exists(out_path):
            continue
        Path(out_path).parent.mkdir(parents=True, exist_ok=True)
        run_model_and_return_samples(args, state, prompt, os.path.join(args.gedit_image_dir, rel))[0].save(out_path)
        done += 1
    print(f"[rank {rank}/{world}] wrote {done} of {len(todo)} assigned images to {args.output_dir}", flush=True)
    D.barrier()
    return done


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("config", type=str)
    ap.add_argument("--pretrained_lvlm_name_or_path", type=str, default=None)
    ap.add_argument("--output_dir", type=str, default=None)
    a = ap.parse_args()
    conf = EvalConfig.from_mapping(yaml.safe_load(Path(a.config).read_text()) or {})
    if a.pretrained_lvlm_name_or_path is not None:
        assert a.output_dir is not None
        conf.pretrained_lvlm_name_or_path, conf.output_dir = a.pretrained_lvlm_name_or_path, a.output_dir
    main(conf)
