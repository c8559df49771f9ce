"""``PipelineMuse``: tokens -> image glue with the reference's call surface (muse/pipeline_muse.py:38-369).

Host-side Python only: it wires ``MaskGitTransformer.generate2`` (fused decode-step kernel) to
``MaskGitVQGAN.decode_code`` (CUDA detokeniser) and converts to PIL.  Class-conditional generation and text
conditioning with *precomputed* ``prompt_embeds`` run fully on the H100 path; raw ``text=`` needs a third-party
text encoder / tokenizer object (CLIP / T5 from ``transformers``), which is outside this repository's scope and is
called as-is when attached -- for ``MaskGiTUViT_v2`` exactly as the reference pipeline calls it (penultimate-layer states,
projected pooled embedding, encoded negative / empty prompt, ``clip_skip``).
"""
from __future__ import annotations

import json
import os
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from .modeling_maskgit_vqgan import MaskGitVQGAN
from .modeling_taming_vqgan import VQGANModel
from .modeling_transformer import MaskGitTransformer
from .modeling_transformer_v2 import MaskGiTUViT_v2
from .sampling import get_mask_chedule


class PipelineMuse:
    def __init__(self, vae, transformer, is_class_conditioned: bool = False, text_encoder=None, tokenizer=None) -> None:
        self.text_encoder = text_encoder
        self.tokenizer = tokenizer
        self.vae = vae
        self.transformer = transformer
        self.is_class_conditioned = is_class_conditioned
        self.device = "cpu"
        self.dtype = torch.float32

    def to(self, device="cpu", dtype=torch.float32):
        self.device, self.dtype = device, dtype
        if not self.is_class_conditioned and self.text_encoder is not None:
            self.text_encoder.to(device, dtype=dtype)
        # master weights stay fp32 on this path (compute is bf16 inside the kernels); the tokenizer is always fp32
        self.transformer.to(device)
        self.vae.to(device, dtype=torch.float32)
        return self

    # -- conditioning ----------------------------------------------------------------------------------------
    def _encode_text(self, text, clip_skip=None):
        if self.text_encoder is None or self.tokenizer is None:
            raise ValueError("text conditioning needs a text_encoder and tokenizer (or pass prompt_embeds=...)")
        ids = self.tokenizer(text, return_tensors="pt", padding="max_length", truncation=True,
                             max_length=self.tokenizer.model_max_length).input_ids.to(self.device)
        return self.text_encoder(ids).last_hidden_state

    def _encode_text_uvit(self, text, negative_text, negative_prompt_embeds, negative_pooled_embeds, clip_skip=None):
        """The text side of the reference pipeline for models with pooled conditioning (muse/pipeline_muse.py:113-197): the
        attached (third-party) CLIP encoder is called as is -- penultimate-layer states (``clip_skip`` picks another layer) and
        the projected pooled embedding for the prompt, layer -2 for the negative prompt, and the encoded empty prompt when
        there is no negative one.  Returns (states, pooled, negative states, negative pooled, (empty states, empty pooled))."""
        if self.text_encoder is None or self.tokenizer is None:
            raise ValueError("MaskGiTUViT_v2 needs prompt_embeds (text states) and pooled_embeds, or a text_encoder and "
                             "tokenizer attached to the pipeline to compute them from `text`")
        if text is None:
            raise ValueError("Either text or class_ids must be provided.")
        text = [text] if isinstance(text, str) else text
        tok = lambda t: self.tokenizer(t, return_tensors="pt", padding="max_length", truncation=True,
                                       max_length=self.tokenizer.model_max_length).input_ids.to(self.device)
        out = self.text_encoder(tok(text), return_dict=True, output_hidden_states=True)
        layer = -(clip_skip + 1) if clip_skip is not None else -2
        pooled, states = out.text_embeds, out.hidden_states[layer]
        empty = (None, None)
        if negative_text is not None:
            neg = [negative_text] * len(text) if isinstance(negative_text, str) else negative_text
            nout = self.text_encoder(tok(neg), return_dict=True, output_hidden_states=True)
            negative_pooled_embeds, negative_prompt_embeds = nout.text_embeds, nout.hidden_states[-2]
        elif negative_prompt_embeds is None:
            ids = self.tokenizer("", padding="max_length", return_tensors="pt").input_ids.to(self.device)
            eout = self.text_encoder(ids, output_hidden_states=True)
            empty = (eout.hidden_states[-2], eout[0])
        return states, pooled, negative_prompt_embeds, negative_pooled_embeds, empty

    @torch.no_grad()
    def __call__(
        self,
        text: Optional[Union[str, List[str]]] = None,
        negative_text: Optional[Union[str, List[str]]] = "",
        prompt_embeds: Optional[torch.Tensor] = None,
        pooled_embeds: Optional[torch.Tensor] = None,
        negative_prompt_embeds: Optional[torch.Tensor] = None,
        negative_pooled_embeds: Optional[torch.Tensor] = None,
        class_ids: Optional[Union[int, List[int]]] = None,
        timesteps: int = 16,
        noise_schedule: str = "cosine",
        guidance_scale: float = 10.0,
        guidance_schedule=None,
        temperature: Union[float, Tuple[float]] = (2, 0),
        topk_filter_thres: float = 0.9,
        num_images_per_prompt: int = 1,
        use_maskgit_generate: bool = True,
        generator: Optional[torch.Generator] = None,
        use_fp16: bool = False,
        noise_type="mask",  # accepted like the reference; only "mask" is implemented
        predict_all_tokens=False,
        orig_size=(512, 512),
        crop_coords=(0, 0),
        aesthetic_score=6.0,
        return_intermediate: bool = False,
        use_tqdm=True,
        transformer_seq_len=None,
        clip_skip: int = None,
        output_type: str = "pil",  # extension: "pt" returns the decoded tensor instead of PIL images
        **unused,
    ):
        if noise_type != "mask" or predict_all_tokens:
            raise NotImplementedError("open_muse_b200.PipelineMuse: only noise_type='mask' without predict_all_tokens")
        if text is None and class_ids is None and prompt_embeds is None:
            raise ValueError("Either text or class_ids must be provided.")
        if text is not None and class_ids is not None:
            raise ValueError("Only one of text or class_ids may be provided.")
        if getattr(self.transformer.config, "add_micro_cond_embeds", False):  # MaskGiTUViT_v2 conditioning (:121-214)
            empty = (None, None)
            if prompt_embeds is None or pooled_embeds is None:  # run the attached text encoder like the reference (:113-197)
                (prompt_embeds, pooled_embeds, negative_prompt_embeds, negative_pooled_embeds,
                 empty) = self._encode_text_uvit(text, negative_text, negative_prompt_embeds, negative_pooled_embeds, clip_skip)
            return self._call_uvit_v2(prompt_embeds, pooled_embeds, negative_prompt_embeds, negative_pooled_embeds, timesteps,
                                      noise_schedule, guidance_scale, guidance_schedule, temperature,
                                      num_images_per_prompt, generator, return_intermediate, output_type, orig_size,
                                      crop_coords, aesthetic_score, transformer_seq_len, empty=empty)
        if return_intermediate:
            raise NotImplementedError("return_intermediate is a MaskGiTUViT_v2.generate2 feature")
        if isinstance(temperature, (tuple, list)):
            temperature = float(temperature[0])  # v1 generate2 takes a scalar that it anneals itself (quirk Q4)
        kwargs = {}
        if class_ids is not None:
            if isinstance(class_ids, int):
                class_ids = [class_ids]
            ids = torch.tensor(class_ids, device=self.device, dtype=torch.long)
            kwargs["class_ids"] = ids.repeat_interleave(num_images_per_prompt, dim=0)
        else:
            if prompt_embeds is None:
                if isinstance(text, str):
                    text = [text]
                prompt_embeds = self._encode_text(text)
                if guidance_scale > 0 and negative_prompt_embeds is None and negative_text is not None:
                    neg = [negative_text] * len(text) if isinstance(negative_text, str) else negative_text
                    negative_prompt_embeds = self._encode_text(neg)
            states = prompt_embeds.to(self.device).repeat_interleave(num_images_per_prompt, dim=0)
            kwargs["encoder_hidden_states"] = states
            if negative_prompt_embeds is not None:
                kwargs["negative_embeds"] = negative_prompt_embeds.to(self.device).repeat_interleave(num_images_per_prompt, dim=0)
            kwargs["guidance_scale"] = guidance_scale
        with torch.autocast("cuda", dtype=torch.bfloat16):
            tokens = self.transformer.generate2(timesteps=timesteps, temperature=temperature, generator=generator,
                                                noise_schedule=get_mask_chedule(noise_schedule), **kwargs)
        return self._decode(tokens, output_type)

    def _decode(self, tokens, output_type):
        """ids -> PIL images (or the fp32 tensor for output_type="pt").  Tokenizers with a fused uint8 path hand back display
        bytes from the device; others go through to_pil_image on the host like the reference."""
        if output_type == "pt":
            return self.vae.decode_code(tokens)
        if hasattr(self.vae, "decode_code_uint8"):
            from PIL import Image

            return [Image.fromarray(a).convert("RGB") for a in self.vae.decode_code_uint8(tokens).cpu().numpy()]
        return [self.to_pil_image(img) for img in self.vae.decode_code(tokens)]

    def _call_uvit_v2(self, prompt_embeds, pooled_embeds, negative_prompt_embeds, negative_pooled_embeds, timesteps,
                      noise_schedule, guidance_scale, guidance_schedule, temperature, num_images_per_prompt, generator,
                      return_intermediate, output_type, orig_size, crop_coords, aesthetic_score, seq_len=None,
                      empty=(None, None)):
        """Text-to-image with ``MaskGiTUViT_v2``: penultimate-layer text states + pooled embedding + micro-conditioning
        (reference pipeline_muse.py:121-233).  The text encoder is third-party and out of scope, so the embeddings (and the
        negative / empty ones needed for guidance) are passed in precomputed."""
        if prompt_embeds is None or pooled_embeds is None:
            raise ValueError("MaskGiTUViT_v2 needs prompt_embeds (text states) and pooled_embeds; run the text encoder "
                             "outside or attach one and encode before calling")
        if guidance_scale > 0 and (negative_prompt_embeds is None or negative_pooled_embeds is None) and empty[0] is None:
            raise ValueError("classifier-free guidance needs negative_prompt_embeds and negative_pooled_embeds (the encoded "
                             "empty prompt)")
        n = num_images_per_prompt
        rep = lambda t: None if t is None else t.to(self.device).repeat_interleave(n, dim=0)
        states, pooled = rep(prompt_embeds), rep(pooled_embeds)
        micro = torch.tensor([list(orig_size) + list(crop_coords) + [aesthetic_score]], device=self.device,
                             dtype=torch.float32)
        if isinstance(temperature, list):
            temperature = tuple(temperature)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = self.transformer.generate2(
                encoder_hidden_states=states, cond_embeds=pooled, micro_conds=micro,
                empty_embeds=None if empty[0] is None else empty[0].to(self.device),
                empty_cond_embeds=None if empty[1] is None else empty[1].to(self.device),
                negative_embeds=rep(negative_prompt_embeds),
                negative_cond_embeds=rep(negative_pooled_embeds), temperature=temperature, timesteps=timesteps,
                guidance_scale=guidance_scale, guidance_schedule=guidance_schedule,
                noise_schedule=get_mask_chedule(noise_schedule), generator=generator,
                return_intermediate=return_intermediate, seq_len=seq_len)
        tokens, intermediate = out if return_intermediate else (out, None)
        images = self._decode(tokens, output_type)
        if return_intermediate:
            inter = [self.vae.decode_code(t) for t in intermediate]
            if output_type != "pt":
                inter = [[self.to_pil_image(img) for img in batch] for batch in inter]
            return images, inter
        return images

    def to_pil_image(self, image: torch.Tensor):
        """[0,1] -> uint8 with the reference's clamp / truncation recipe (pipeline_muse.py:245-252, quirk Q10)."""
        from PIL import Image

        x = image.permute(1, 2, 0).float().cpu().numpy()
        x = (np.clip(2.0 * x - 1.0, -1.0, 1.0) + 1.0) / 2.0
        return Image.fromarray((255 * x).astype(np.uint8)).convert("RGB")

    # -- persistence: <dir>/{vae,transformer}[/text_encoder] like the reference (:254-369) ---------------------
    def save_pretrained(self, save_directory: str) -> None:
        self.vae.save_pretrained(os.path.join(save_directory, "vae"))
        self.transformer.save_pretrained(os.path.join(save_directory, "transformer"))
        if self.text_encoder is not None:
            self.text_encoder.save_pretrained(os.path.join(save_directory, "text_encoder"))
            self.tokenizer.save_pretrained(os.path.join(save_directory, "text_encoder"))

    @classmethod
    def from_pretrained(cls, model_name_or_path: str = None, text_encoder_path: Optional[str] = None,
                        vae_path: Optional[str] = None, transformer_path: Optional[str] = None, vae=None,
                        text_encoder=None, transformer=None, is_class_conditioned: bool = False):
        if model_name_or_path is None and (vae_path is None or transformer_path is None):
            raise ValueError("If model_name_or_path is None, then text_encoder_path, vae_path, and transformer_path must be provided.")

        def sub(path, name):
            return (path, None) if model_name_or_path is None else (model_name_or_path, name)

        def class_name(path, subfolder):
            p = os.path.join(path, subfolder, "config.json") if subfolder else os.path.join(path, "config.json")
            return json.load(open(p))["_class_name"] if os.path.isfile(p) else None

        if vae is None:
            path, folder = sub(vae_path, "vae")
            name = class_name(path, folder)
            if name == "VQGANModel":  # (reference :327-328)
                vae = VQGANModel.from_pretrained(path, subfolder=folder)
            elif name in (None, "MaskGitVQGAN"):
                vae = MaskGitVQGAN.from_pretrained(path, subfolder=folder)
            else:
                raise NotImplementedError(f"tokenizer class {name} is out of scope (MaskGitVQGAN and VQGANModel are built)")
        if transformer is None:
            path, folder = sub(transformer_path, "transformer")
            name = class_name(path, folder)
            if name in ("MaskGiTUViT", "MaskGiTUViT_v2"):  # (reference :317-318)
                transformer = MaskGiTUViT_v2.from_pretrained(path, subfolder=folder)
            elif name in (None, "MaskGitTransformer"):
                transformer = MaskGitTransformer.from_pretrained(path, subfolder=folder)
            else:
                raise ValueError(f"Unknown Transformer class: {name}")
        tokenizer = None
        if not is_class_conditioned:  # (reference :298-314: the tokenizer is always loaded, the encoder unless one was passed)
            path, folder = sub(text_encoder_path, "text_encoder")
            from transformers import AutoTokenizer, CLIPTextModel, CLIPTextModelWithProjection, T5EncoderModel

            full = os.path.join(path, folder) if folder else path
            if text_encoder is None:
                if getattr(transformer.config, "add_cond_embeds", False):
                    # models with pooled conditioning (MaskGiTUViT_v2): upstream loads CLIPTextModelWithProjection
                    # unconditionally -- the only class whose outputs carry text_embeds
                    enc_cls = CLIPTextModelWithProjection
                else:  # v1 transformers read last_hidden_state only (upstream's pipeline cannot drive them, quirk Q15)
                    enc_cls = CLIPTextModel if "clip" in str(full).lower() else T5EncoderModel
                text_encoder = enc_cls.from_pretrained(full)
            tokenizer = AutoTokenizer.from_pretrained(full)
        return cls(vae=vae, transformer=transformer, is_class_conditioned=is_class_conditioned,
                   text_encoder=text_encoder, tokenizer=tokenizer)


class PipelineMuseInpainting(PipelineMuse):
    """Masked-region regeneration (muse/pipeline_muse.py:372-512): tokenise the image, overwrite the masked token
    positions with the mask id and let ``generate2`` fill them in; known tokens are kept by the fused decode step."""

    def _inpaint_uvit_v2(self, image_tokens, text, negative_text, timesteps, guidance_scale, guidance_schedule, temperature,
                         n, generator, orig_size, crop_coords, aesthetic_score, output_type):
        """Text-conditioned inpainting with ``MaskGiTUViT_v2`` through the attached text encoder, as the reference wires it
        (:424-498): penultimate-layer states + pooled embedding for the prompt, the LAST layer for an explicit negative prompt
        (upstream's choice here, unlike PipelineMuse), the encoded empty prompt always passed along, micro-conditioning; the
        start tokens keep their own length while ``seq_len`` stays at generate2's default of 256 for the mask schedule."""
        if self.text_encoder is None or self.tokenizer is None or text is None:
            raise ValueError("PipelineMuseInpainting with MaskGiTUViT_v2 needs `text` and an attached text_encoder / tokenizer")
        text = [text] if isinstance(text, str) else text
        tok = lambda t: self.tokenizer(t, return_tensors="pt", padding="max_length", truncation=True,
                                       max_length=self.tokenizer.model_max_length).input_ids.to(self.device)
        pooled = None
        if getattr(self.transformer.config, "add_cond_embeds", False):
            out = self.text_encoder(tok(text), return_dict=True, output_hidden_states=True)
            pooled, states = out.text_embeds, out.hidden_states[-2]
        else:
            states = self.text_encoder(tok(text)).last_hidden_state
        neg = None
        if negative_text is not None:
            neg = self.text_encoder(tok([negative_text] if isinstance(negative_text, str) else negative_text)).last_hidden_state
        rep = lambda t: None if t is None else t.repeat_interleave(n, dim=0)
        ids = self.tokenizer("", padding="max_length", return_tensors="pt").input_ids.to(self.device)
        eout = self.text_encoder(ids, output_hidden_states=True)
        micro = torch.tensor([list(orig_size) + list(crop_coords) + [aesthetic_score]], device=self.device, dtype=states.dtype)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            tokens = self.transformer.generate2(
                input_ids=image_tokens, encoder_hidden_states=rep(states), negative_embeds=rep(neg),
                empty_embeds=eout.hidden_states[-2], empty_cond_embeds=eout[0], cond_embeds=rep(pooled), micro_conds=micro,
                timesteps=timesteps, guidance_scale=guidance_scale, guidance_schedule=guidance_schedule,
                temperature=temperature, generator=generator)
        return self._decode(tokens, output_type)

    @staticmethod
    def _to_pixel_values(image, image_size):
        """Resize(shorter side, bilinear) -> CenterCrop -> ToTensor of the reference (:404-410), without torchvision."""
        if isinstance(image, torch.Tensor):
            return image if image.dim() == 4 else image.unsqueeze(0)
        from PIL import Image

        w, h = image.size
        if w <= h:
            nw, nh = image_size, int(image_size * h / w)
        else:
            nw, nh = int(image_size * w / h), image_size
        image = image.convert("RGB").resize((nw, nh), Image.BILINEAR)
        left, top = int(round((nw - image_size) / 2.0)), int(round((nh - image_size) / 2.0))
        image = image.crop((left, top, left + image_size, top + image_size))
        x = torch.from_numpy(np.asarray(image, dtype=np.uint8).copy()).permute(2, 0, 1).float().div_(255.0)
        return x.unsqueeze(0)

    @torch.no_grad()
    def __call__(
        self,
        image,
        mask: torch.BoolTensor,
        text: Optional[Union[str, List[str]]] = None,
        negative_text: Optional[Union[str, List[str]]] = None,
        class_ids: torch.LongTensor = None,
        timesteps: int = 8,
        guidance_scale: float = 8.0,
        guidance_schedule=None,
        temperature: float = 1.0,
        topk_filter_thres: float = 0.9,
        num_images_per_prompt: int = 1,
        use_maskgit_generate: bool = True,
        generator: Optional[torch.Generator] = None,
        use_fp16: bool = False,
        image_size: int = 256,
        orig_size=(256, 256),
        crop_coords=(0, 0),
        aesthetic_score=6.0,
        prompt_embeds: Optional[torch.Tensor] = None,
        negative_prompt_embeds: Optional[torch.Tensor] = None,
        output_type: str = "pil",
    ):
        assert use_maskgit_generate
        if text is None and class_ids is None and prompt_embeds is None:
            raise ValueError("Either text or class_ids must be provided.")
        if text is not None and class_ids is not None:
            raise ValueError("Only one of text or class_ids may be provided.")
        pixel_values = self._to_pixel_values(image, image_size).to(self.device)
        _, image_tokens = self.vae.encode(pixel_values)
        image_tokens[mask.to(image_tokens.device).reshape(1, -1).expand_as(image_tokens)] = self.transformer.config.mask_token_id
        image_tokens = image_tokens.repeat(num_images_per_prompt, 1)
        if getattr(self.transformer.config, "add_micro_cond_embeds", False) and class_ids is None:
            return self._inpaint_uvit_v2(image_tokens, text, negative_text, timesteps, guidance_scale, guidance_schedule,
                                         temperature, num_images_per_prompt, generator, orig_size, crop_coords,
                                         aesthetic_score, output_type)
        kwargs = {}
        if class_ids is not None:
            if isinstance(class_ids, int):
                class_ids = [class_ids]
            ids = torch.as_tensor(class_ids, device=self.device, dtype=torch.long)
            kwargs["class_ids"] = ids.repeat_interleave(num_images_per_prompt, dim=0)
        else:
            if prompt_embeds is None:
                text = [text] if isinstance(text, str) else text
                prompt_embeds = self._encode_text(text)
                if negative_text is not None and negative_prompt_embeds is None:
                    neg = [negative_text] if isinstance(negative_text, str) else negative_text
                    negative_prompt_embeds = self._encode_text(neg)
            kwargs["encoder_hidden_states"] = prompt_embeds.to(self.device).repeat_interleave(num_images_per_prompt, dim=0)
            if negative_prompt_embeds is not None:
                kwargs["negative_embeds"] = negative_prompt_embeds.to(self.device).repeat_interleave(num_images_per_prompt, dim=0)
            kwargs["guidance_scale"] = guidance_scale
        with torch.autocast("cuda", dtype=torch.bfloat16):
            tokens = self.transformer.generate2(input_ids=image_tokens, timesteps=timesteps, temperature=temperature,
                                                generator=generator, **kwargs)
        return self._decode(tokens, output_type)
