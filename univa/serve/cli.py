"""`python -m univa.serve.cli` — the reference's serving entry point (univa/serve/cli.py:118-286)
over the libb2f engine: same flags (`--model_path --flux_path --height --width --num_inference_steps
--guidance_scale --no_joint_with_t5 --ocr_enhancer --no_auto_hw`), same turn structure
(VLM prefill -> task head -> MLP2 -> [T5 ‖ CLIP] -> FluxKontextPipeline -> PNG).

The prompt path is the reference's (cli.py:131-198): a running `conversation` of chat messages and
`history_image_paths`, `processor.apply_chat_template(..., add_generation_prompt=True)` with the system turn
dropped, `process_vision_info` (448x448-pixel budget per image, aspect ratio kept), `processor(text=, images=)`;
the processor (tokenizer + image processor + chat template) is loaded from `--model_path` and its absence is an
error.  Text replies are decoded with `processor.batch_decode` (cli.py:261-263).

Differences, all forced by this environment and all explicit:
  * `--synthetic` builds every model with seeded random weights at the real architecture sizes (no
    checkpoints or tokenizer files exist offline); ONLY then do token ids follow SURVEY.md §8d's canonical
    layout instead of the chat template.  Without `--synthetic` the loaders in
    gpt_image_edit_b200.checkpoint read the reference's checkpoint directories (safetensors) and the
    processor files next to them.
  * one VLM prefill per turn instead of the reference's two identical ones (cli.py:200 and :211):
    `hidden_states[-1]` of the first equals the pre-MLP2 tensor of the second.
  * with `--synthetic` the T5-XXL / CLIP-L encoders carry seeded random weights and the prompt is
    tokenised by `SyntheticTokenizer` (no vocabulary files offline); the text-reply branch
    (`model.generate`, greedy KV-cache decode) prints token ids when no tokenizer files are available.
  * `--prompt/--image/--output` run one non-interactive turn (the reference is REPL-only).
"""
from __future__ import annotations

import argparse

import numpy as np
import torch

from gpt_image_edit_b200 import ops
from gpt_image_edit_b200._lib import B2FError
from gpt_image_edit_b200.image_io import image_to_condition_tensor, process_vision_info, qwen_pixel_values, resize_u8
from gpt_image_edit_b200.pipeline import FluxKontextPipeline
from gpt_image_edit_b200.scheduler import FlowMatchEulerDiscreteScheduler
from gpt_image_edit_b200.text_encoders import (B200CLIPTextModel, B200T5Encoder, CLIPTextConfig, SyntheticTokenizer,
                                               T5EncoderConfig, encode_prompt)
from gpt_image_edit_b200.vae import B200AutoencoderKL
from univa.models.qwen2p5vl.modeling_univa_qwen2p5vl import UnivaQwen2p5VLConfig, UnivaQwen2p5VLForConditionalGeneration
from univa.utils.anyres_util import dynamic_resize

seed = 42
generate_image_temp = "./generate_image_{}.png"          # reference cli.py:27
ASSISTANT_TOKEN_ID = 77091          # reference cli.py:202
IM_START, IM_END, VISION_START, VISION_END, IMAGE_PAD = 151644, 151645, 151652, 151653, 151655


class TaskHead(torch.nn.Module):
    """Linear(3584,10240)·SiLU·Dropout·Linear(10240,2) (reference cli.py:42-49) as two libb2f GEMMs."""

    def __init__(self, hidden=3584, inner=10240, device="cuda"):
        super().__init__()
        z = lambda *s: torch.zeros(s, device=device, dtype=torch.bfloat16)
        self.w0, self.b0, self.w3, self.b3 = z(inner, hidden), z(inner), z(8, inner), z(8)   # 2 logits, rows padded to 8

    @torch.no_grad()
    def forward(self, x):
        return ops.linear(ops.linear(x.to(torch.bfloat16), self.w0, self.b0, epilogue=ops.EPI_SILU), self.w3, self.b3)[:, :2]


def load_main_model_and_processor(model_path, device, synthetic=False, small=False, min_pixels=448 * 448,
                                  max_pixels=448 * 448, task_head: bool = True, **config_overrides):
    """-> (model, task_head, processor)  (reference cli.py:30-56).  processor is None only with --synthetic;
    `task_head=False` (eval drivers, training) does not read `task_head_final.pt`."""
    if not synthetic:
        from gpt_image_edit_b200.checkpoint import load_univa_checkpoint
        return load_univa_checkpoint(model_path, device, min_pixels=min_pixels, max_pixels=max_pixels, task_head=task_head)
    kw = {}
    if small:  # plumbing runs: a few layers at full width
        kw = dict(text_config=dict(num_hidden_layers=2), vision_config=dict(depth=2, fullatt_block_indexes=(1,)),
                  denoise_tower=dict(denoiser_config=dict(num_layers=1, num_single_layers=1)))
    kw.update(config_overrides)     # e.g. the special-token ids of a non-Qwen tokenizer (tests)
    cfg = UnivaQwen2p5VLConfig(**kw)
    model = UnivaQwen2p5VLForConditionalGeneration(cfg, device=device)
    model.lvlm.randomize_(seed=10)
    model.denoise_tower.denoiser.randomize_(seed=0)
    g = torch.Generator(device=device).manual_seed(11)
    for t in model.denoise_tower.denoise_projector.state_dict().values():
        t.copy_((torch.randn(t.shape, device=device, generator=g) * 0.02).to(torch.bfloat16))
    head = TaskHead(cfg.hidden_size, device=device)
    head.w0.copy_((torch.randn(head.w0.shape, device=device, generator=g) * 0.02).to(torch.bfloat16))
    head.w3[:2].copy_((torch.randn(2, head.w3.shape[1], device=device, generator=g) * 0.02).to(torch.bfloat16))
    head.b3[1] = 1.0   # synthetic head always routes to "generate"
    return model, head, None


def load_pipe(denoiser, flux_path, device, synthetic=False, small=False):
    """-> (pipe, [clip_tokenizer, t5_tokenizer], [clip, t5])  (reference cli.py:58-76)."""
    if not synthetic:
        pipe = FluxKontextPipeline.from_pretrained(flux_path, transformer=denoiser, torch_dtype=torch.bfloat16)
    else:
        vae = B200AutoencoderKL(device=device).randomize_(seed=1)
        ccfg = CLIPTextConfig(num_hidden_layers=2) if small else CLIPTextConfig()
        tcfg = T5EncoderConfig(num_layers=1) if small else T5EncoderConfig()
        pipe = FluxKontextPipeline(transformer=denoiser, vae=vae, scheduler=FlowMatchEulerDiscreteScheduler(),
                                   text_encoder=B200CLIPTextModel(ccfg, device=device).randomize_(seed=20),
                                   tokenizer=SyntheticTokenizer.clip(ccfg.vocab_size),
                                   text_encoder_2=B200T5Encoder(tcfg, device=device).randomize_(seed=21),
                                   tokenizer_2=SyntheticTokenizer.t5(tcfg.vocab_size))
    return pipe, [pipe.tokenizer, pipe.tokenizer_2], [pipe.text_encoder, pipe.text_encoder_2]


def update_size(shapes, anyres="any_11ratio", anchor_pixels=1024 * 1024):
    """(h, w) of the generation from the input image sizes (reference cli.py:82-97)."""
    if not shapes:
        return int(anchor_pixels ** 0.5), int(anchor_pixels ** 0.5)
    w = sum(s[0] for s in shapes) / len(shapes)
    h = sum(s[1] for s in shapes) / len(shapes)
    return dynamic_resize(int(h), int(w), anyres, anchor_pixels=anchor_pixels)


def synthetic_chat_tokens(n_image_tokens: int, n_text: int = 24, vocab: int = 152064, seed_: int = 2):
    """<|im_start|> user \\n <|vision_start|> [image_pad]*n <|vision_end|> text... <|im_end|> \\n <|im_start|> assistant \\n
    with seeded text ids (the chat template needs tokenizer files that are not available offline)."""
    g = torch.Generator().manual_seed(seed_)
    text = torch.randint(1000, 100000, (n_text,), generator=g).tolist()
    ids = [IM_START, 872, 198, VISION_START] + [IMAGE_PAD] * n_image_tokens + [VISION_END] + text + \
          [IM_END, 198, IM_START, ASSISTANT_TOKEN_ID, 198]
    return torch.tensor([ids])


def prepare_inputs(processor, conversation, device):
    """Chat messages -> model inputs, as the reference does it (cli.py:183-198; gedit/step1_gen_samples.py:136-151):
    chat template with the generation prompt, the default system turn dropped, images fetched and resized by
    `process_vision_info`, then the processor call that expands `<|image_pad|>` and builds pixel_values."""
    chat_text = processor.apply_chat_template(conversation, tokenize=False, add_generation_prompt=True)
    chat_text = "<|im_end|>\n".join(chat_text.split("<|im_end|>\n")[1:])   # drop system
    image_inputs, video_inputs = process_vision_info(conversation)
    inputs = processor(text=[chat_text], images=image_inputs, videos=video_inputs, padding=True, return_tensors="pt")
    return inputs.to(device)


def prepare_condition_images(image_paths, device):
    """[-1, 1] float32 [N, 3, H, W] of the history images (reference cli.py:99-116)."""
    from PIL import Image

    if not image_paths:
        return None
    imgs = [image_to_condition_tensor(np.asarray(Image.open(p).convert("RGB")))[0] for p in image_paths]
    return torch.stack(imgs).to(device, dtype=torch.float32)


class ChatSession:
    """State of the reference's REPL (cli.py:131-137): `conversation`, `history_image_paths`, output counter."""

    def __init__(self, args, model, task_head, pipe, processor, tokenizers, text_encoders, device):
        self.args, self.model, self.task_head, self.pipe, self.processor = args, model, task_head, pipe, processor
        self.tokenizers, self.text_encoders, self.device = tokenizers, text_encoders, device
        self.conversation: list = []
        self.history_image_paths: list = []
        self.cur_genimg_i = 0
        if processor is None and not getattr(args, "synthetic", False):
            raise B2FError("no processor (tokenizer / chat template / image processor files) was found under --model_path; "
                           "the instruction cannot reach the VLM without it.  Pass --synthetic for the offline plumbing run")

    # ------------------------------------------------------------------ prompt construction (cli.py:151-197)
    def add_user_turn(self, txt: str, urls: list):
        """Append the user's message (text, then one image item per url with the 448x448-pixel budget) to the
        conversation and the urls to the image history; -> (height, width) of the generation."""
        args = self.args
        from PIL import Image

        content = []
        if txt:
            if getattr(args, "ocr_enhancer", False) and urls:
                raise B2FError("--ocr_enhancer needs the paddleocr service of the reference (univa/utils/get_ocr.py): out of scope")
            content.append({"type": "text", "text": txt})
        new_h, new_w = args.height, args.width
        if urls:
            for url in urls:
                content.append({"type": "image", "image": url, "min_pixels": 448 * 448, "max_pixels": 448 * 448})
                self.history_image_paths.append(url)
            # the reference calls update_size whenever the turn has images; its --no_auto_hw flag is parsed but unused
            shapes = [Image.open(u).size for u in urls[:2]]
            new_h, new_w = update_size(shapes, "any_11ratio", anchor_pixels=args.height * args.width)
        self.conversation.append({"role": "user", "content": content})
        return new_h, new_w

    def model_inputs(self):
        """(input_ids, attention_mask, pixel_values | None, image_grid_thw | None) for the whole conversation."""
        dev = self.device
        if self.processor is not None:
            inputs = prepare_inputs(self.processor, self.conversation, dev)
            has_img = "pixel_values" in inputs
            return (inputs["input_ids"], inputs["attention_mask"], inputs["pixel_values"] if has_img else None,
                    inputs["image_grid_thw"] if has_img else None)
        # --synthetic: canonical token layout (SURVEY.md section 8d), one 448x448 view of the latest image
        from PIL import Image

        pixel_values = grid = None
        n_img_tok = 0
        if self.history_image_paths:
            img = np.asarray(Image.open(self.history_image_paths[-1]).convert("RGB"))
            pixel_values, grid = qwen_pixel_values(resize_u8(img, 448, 448))
            pixel_values = pixel_values.to(dev)
            n_img_tok = pixel_values.shape[0] // 4
        input_ids = synthetic_chat_tokens(n_img_tok).to(dev)
        return input_ids, torch.ones_like(input_ids), pixel_values, grid

    # ------------------------------------------------------------------ one turn (cli.py:139-267)
    @torch.no_grad()
    def turn(self, txt: str, urls: list, output_path: str | None = None):
        """-> ("image", path) or ("text", reply)"""
        args, dev = self.args, self.device
        new_h, new_w = self.add_user_turn(txt, urls)
        input_ids, attention_mask, pixel_values, grid = self.model_inputs()

        hidden = self.model.prefill_hidden(input_ids, pixel_values=pixel_values, attention_mask=attention_mask,
                                           image_grid_thw=grid)
        assistant_vec = hidden[input_ids == ASSISTANT_TOKEN_ID][-1:]
        if assistant_vec.shape[0] == 0:
            raise B2FError(f"token id {ASSISTANT_TOKEN_ID} ('assistant') does not occur in the prompt: the tokenizer under "
                           "--model_path is not the Qwen2.5-VL tokenizer the task head was trained with")
        task = self.task_head(assistant_vec)[0].float()
        if getattr(args, "force_text_reply", False):
            task = torch.tensor([1.0, 0.0])
        if not (task[0] < task[1]):
            # understanding branch (cli.py:256-267): greedy KV-cache decode, reply = the newly generated ids
            generated = self.model.generate(input_ids=input_ids, pixel_values=pixel_values, attention_mask=attention_mask,
                                            image_grid_thw=grid, max_new_tokens=args.max_new_tokens)
            reply = reply_text(generated[0, input_ids.shape[1]:].tolist(), self.processor)
            self.conversation.append({"role": "assistant", "content": [{"type": "text", "text": reply}]})
            return "text", reply
        lvlm_embeds = self.model.denoise_tower.denoise_projector(hidden)                 # MLP2 -> [1, L, 4096]
        assert lvlm_embeds.shape[0] == 1
        # [T5 ‖ CLIP] on the libb2f encoders; an empty T5 prompt under --no_joint_with_t5 (cli.py:221-234)
        t5_embeds, pooled = encode_prompt(self.text_encoders, self.tokenizers, txt if not args.no_joint_with_t5 else "", 256,
                                          dev, 1)
        prompt_embeds = lvlm_embeds if args.no_joint_with_t5 else torch.cat([lvlm_embeds, t5_embeds], dim=1)
        if len(self.history_image_paths) > 1:
            # the reference stacks every history image into `image=` (cli.py:237) and its prepare_latents then fails on the
            # batch mismatch (flux_pipeline.py:676-690 keep N latents for batch 1): one context image per session
            raise B2FError("more than one image in the session history: the reference pipeline accepts a single context image "
                           "per edit (start a new session to edit a generated image)")
        cond = prepare_condition_images(self.history_image_paths, dev)
        image = self.pipe(image=cond, prompt_embeds=prompt_embeds, pooled_prompt_embeds=pooled, height=new_h, width=new_w,
                          num_inference_steps=args.num_inference_steps, guidance_scale=args.guidance_scale,
                          generator=torch.Generator(device=dev).manual_seed(seed),
                          **({"max_area": args.max_area, "_auto_resize": False} if args.max_area else {})).images[0]
        img_url = output_path or generate_image_temp.format(self.cur_genimg_i)
        self.cur_genimg_i += 1
        image.save(img_url)
        self.conversation.append({"role": "assistant", "content": [{"type": "image", "image": img_url}]})
        self.history_image_paths.append(img_url)
        return "image", img_url


def reply_text(token_ids, processor=None):
    """Decoded reply when a processor / tokenizer is available (reference cli.py:261-263), else the raw ids."""
    if processor is not None:
        return processor.batch_decode([token_ids], skip_special_tokens=True, clean_up_tokenization_spaces=False)[0]
    return "<token ids> " + " ".join(str(t) for t in token_ids)


def main(args):
    if not torch.cuda.is_available():
        raise SystemExit("univa.serve.cli runs on an H100 through libb2f; there is no CPU path")
    device = torch.device("cuda")
    model, task_head, processor = load_main_model_and_processor(args.model_path, device, args.synthetic, args.small)
    pipe, tokenizers, text_encoders = load_pipe(model.denoise_tower.denoiser, args.flux_path, device, args.synthetic, args.small)
    if getattr(args, "fp8", False) or getattr(args, "fp8_attention", False):
        pipe.transformer.enable_fp8(linears=getattr(args, "fp8", False), attention=getattr(args, "fp8_attention", False))
    if getattr(args, "cache_threshold", None) is not None:
        from gpt_image_edit_b200.flux_transformer import FirstBlockCacheConfig
        pipe.transformer.enable_cache(FirstBlockCacheConfig(threshold=args.cache_threshold))
    session = ChatSession(args, model, task_head, pipe, processor, tokenizers, text_encoders, device)

    if args.prompt is not None or args.image is not None:       # one non-interactive turn
        kind, out = session.turn(args.prompt or "", [args.image] if args.image else [], output_path=args.output)
        print(f"Assistant: generate image at {out}" if kind == "image" else f"Assistant: {out}")
        return
    print("Interactive UniWorld-V1 Chat (Exit if input is empty)")
    while True:
        txt = input("Text prompt (or press Enter to skip): ").strip()
        img_input = input("Image URLs (comma-separated, or press Enter to skip): ").strip()
        if not img_input and not txt:
            print("Exit.")
            break
        urls = [u.strip() for u in img_input.split(",") if u.strip()]
        kind, out = session.turn(txt, urls)
        print(f"Assistant: generate image at {out}\n" if kind == "image" else f"Assistant: {out}\n")


def build_parser():
    p = argparse.ArgumentParser(description="Model and component paths")
    p.add_argument("--model_path", type=str, default="")
    p.add_argument("--flux_path", type=str, default="")
    p.add_argument("--no_auto_hw", action="store_true")
    p.add_argument("--height", type=int, default=1024)
    p.add_argument("--width", type=int, default=1024)
    p.add_argument("--num_inference_steps", type=int, default=28)
    p.add_argument("--guidance_scale", type=float, default=3.5)
    p.add_argument("--ocr_enhancer", action="store_true")
    p.add_argument("--no_joint_with_t5", action="store_true")
    # additions
    p.add_argument("--synthetic", action="store_true", help="seeded random weights (no checkpoints offline)")
    p.add_argument("--small", action="store_true", help="with --synthetic: a few layers only (plumbing runs)")
    p.add_argument("--max_area", type=int, default=0, help="pass max_area to the pipeline and disable _auto_resize "
                   "(the reference always rescales to ~1 MP, SURVEY.md §0 item 8)")
    p.add_argument("--max_new_tokens", type=int, default=128, help="text-reply branch (reference: 128)")
    p.add_argument("--force_text_reply", action="store_true", help="with --synthetic: route the turn to the text-reply "
                   "branch (the synthetic task head otherwise always chooses 'generate image')")
    p.add_argument("--fp8", action="store_true", help="run the denoiser's block linears in FP8 (e4m3 tensor cores, "
                   "per-token / per-channel scales; adds an 8.6 GB e4m3 copy of those weights)")
    p.add_argument("--fp8-attention", action="store_true", help="run the denoiser's joint attention in FP8 (e4m3 "
                   "tensor cores, per-head Q / K and per-channel V scales); combines with --fp8.  Faster, but heads "
                   "with peaked attention lose accuracy (e4m3 scores: about 13%% rel-L2 on peaked synthetic heads, "
                   "against 0.2%% in bf16), which can show in the image")
    p.add_argument("--cache-threshold", type=float, default=None, help="first-block cache of the denoiser (off when "
                   "absent): skip blocks 1.. on steps whose block-0 residual moved by less than this relative L1 "
                   "distance since the last full step.  An approximation; its effect on images depends on the checkpoint")
    p.add_argument("--prompt", type=str, default=None)
    p.add_argument("--image", type=str, default=None)
    p.add_argument("--output", type=str, default="output.png")
    return p


if __name__ == "__main__":
    a = build_parser().parse_args()
    if not a.synthetic and not (a.model_path and a.flux_path):
        raise SystemExit("--model_path and --flux_path are required (or pass --synthetic)")
    main(a)
