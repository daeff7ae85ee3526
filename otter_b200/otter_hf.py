"""HF-level boundary: OtterConfig, OtterPreTrainedModel, OtterModel, OtterForConditionalGeneration.

Mirrors the public surface of /root/reference/src/otter_ai/models/otter/modeling_otter.py:523-1042 and
configuration_otter.py — constructor, forward()/generate()/_encode_vision_x signatures, attribute names,
freeze policy, assertion / error behaviour — while the vision-fusion hot path (CLIP -> perceiver -> gated
cross-attention) runs on the otter_b200 kernels.  The frozen language model is stock code (HF LLaMA; the
reference's own MPT / MosaicGPT / Falcon classes when the reference package is importable): it is outside the
hot path (SURVEY.md §8f).
"""
import copy
import os
from typing import List, Optional

import torch
import torch.nn as nn
from transformers.configuration_utils import PretrainedConfig
from transformers.modeling_outputs import CausalLMOutputWithPast
from transformers.modeling_utils import PreTrainedModel
from transformers.models.auto import CONFIG_MAPPING, AutoTokenizer
from transformers.models.clip import CLIPVisionConfig

from .modeling_clip import CLIPVisionModel
from .modeling_otter import (OtterLMMixin, OtterPerceiverResampler, _infer_decoder_layers_attr_name, encode_vision_x,
                             extend_instance)


def master_print(*args, **kwargs):
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_rank() != 0:
        return
    print(*args, **kwargs)


def _reference_lm(arch):
    """MPT: otter_b200.lm_mpt.  MosaicGPT / Falcon live in the reference package (frozen LMs, out of scope here)."""
    if arch == "MPTForCausalLM":      # this repo's own MPT on the otter_b200 kernels (SURVEY.md 8f rank 1)
        from .lm_mpt import MPTConfig, MPTForCausalLM
        return MPTConfig, MPTForCausalLM, "mosaicml/mpt-7b-instruct"
    try:
        if arch == "MosaicGPT":
            from otter_ai.models.mpt_redpajama.configuration_mosaic_gpt import MosaicGPTConfig
            from otter_ai.models.mpt_redpajama.mosaic_gpt import MosaicGPT
            return MosaicGPTConfig, MosaicGPT, "mosaicml/mosaic-llama-redpajama-final-candidate"
        if arch == "RWForCausalLM":
            from otter_ai.models.falcon.configuration_RW import RWConfig
            from otter_ai.models.falcon.modelling_RW import RWForCausalLM
            return RWConfig, RWForCausalLM, "PATH-TO-YOUR-FALCON"
    except ImportError as e:
        raise ImportError(f"text architecture {arch} needs the reference's `otter_ai` package on sys.path "
                          f"(its frozen LM is reused unchanged): {e}") from e
    raise ValueError(f"unsupported text architecture {arch}")


class OtterConfig(PretrainedConfig):
    """configuration_otter.py:15-97 — vision_config (CLIP), text_config (dispatched on architectures[0])."""
    model_type = "otter"
    is_composition = True

    def __init__(self, vision_config=None, text_config=None, cross_attn_every_n_layers: int = 4,
                 use_media_placement_augmentation: bool = True, **kwargs):
        super().__init__(**kwargs)
        vision_config = dict(vision_config or {})
        text_config = dict(text_config or {})
        self.vision_config = CLIPVisionConfig(**vision_config)
        arch = (text_config.get("architectures") or [None])[0]
        if arch in ("MPTForCausalLM", "MosaicGPT", "RWForCausalLM"):
            self.text_config = _reference_lm(arch)[0](**text_config)
        elif text_config:
            self.text_config = CONFIG_MAPPING[text_config.pop("model_type")](**text_config)
        else:
            self.text_config = CONFIG_MAPPING["llama"]()
        self.cross_attn_every_n_layers = cross_attn_every_n_layers
        self.use_media_placement_augmentation = use_media_placement_augmentation

    def to_dict(self):
        output = copy.deepcopy(self.__dict__)
        output["vision_config"] = self.vision_config.to_dict()
        output["text_config"] = self.text_config.to_dict()
        output["model_type"] = self.__class__.model_type
        return output


class OtterPreTrainedModel(PreTrainedModel):
    config_class = OtterConfig
    base_model_prefix = "otter"
    supports_gradient_checkpointing = True
    _no_split_modules = ["OtterPerceiverBlock", "CLIPEncoderLayer", "OtterLayer", "CLIPVisionModel"]

    def _init_weights(self, module):
        """Otter requires no specific initialization (reference :534-536)."""
        return None


def _build_lang_encoder(text_config):
    name = getattr(text_config, "_name_or_path", "") or ""
    arch = (getattr(text_config, "architectures", None) or ["LlamaForCausalLM"])[0]
    if "llama" in name or arch == "LlamaForCausalLM":
        from transformers import LlamaForCausalLM
        from . import lm_llama
        lm = LlamaForCausalLM(config=text_config)
        if os.environ.get("OTB_LLAMA_LAYERS", "1") != "0" and lm_llama.swappable(text_config):
            lm_llama.swap_llama_layers(lm)     # frozen decoder layers on the otter_b200 kernels (SURVEY.md 8f rank 1)
        return lm, name
    _, cls, tok = _reference_lm(arch)
    return cls(config=text_config), tok


class _OtterBase(OtterPreTrainedModel):
    """Construction shared by OtterModel (:539-736) and OtterForConditionalGeneration (:739-1042)."""
    _resize_llama_embeddings = False
    _special_tokens = ["<|endofchunk|>", "<image>", "<answer>"]
    _honour_media_placement_augmentation = False    # Otter forces it off (:786); Flamingo reads the config
    _use_frame_embs = True                          # Flamingo builds its perceiver without frame_embs
    _assert_single_frame = False
    _perceiver_cls = OtterPerceiverResampler
    _lm_mixin_cls = OtterLMMixin

    def __init__(self, config: OtterConfig):
        super().__init__(config)
        lang_encoder, tok_name = _build_lang_encoder(config.text_config)
        text_tokenizer = AutoTokenizer.from_pretrained(tok_name)
        text_tokenizer.add_special_tokens({"additional_special_tokens": list(self._special_tokens)})
        if text_tokenizer.pad_token is None:
            text_tokenizer.add_special_tokens({"pad_token": "<PAD>"})
        self.text_tokenizer = text_tokenizer
        self.eoc_token_id = text_tokenizer.encode("<|endofchunk|>")[-1]
        self.media_token_id = text_tokenizer.encode("<image>")[-1]

        extend_instance(lang_encoder, self._lm_mixin_cls)
        lang_encoder.set_decoder_layers_attr_name(_infer_decoder_layers_attr_name(lang_encoder))
        if self._resize_llama_embeddings and lang_encoder.__class__.__name__ == "LlamaForCausalLM":
            lang_encoder.resize_token_embeddings(len(text_tokenizer))
        self.lang_encoder = lang_encoder

        self.cross_attn_every_n_layers = config.cross_attn_every_n_layers
        self.use_media_placement_augmentation = (bool(config.use_media_placement_augmentation)
                                                 if self._honour_media_placement_augmentation else False)
        self.max_num_frames = (config.max_num_frames if hasattr(config, "max_num_frames") else None) \
            if self._use_frame_embs else None
        if self._use_frame_embs:
            kind = "Otter-Image" if self.max_num_frames in (None, 1) else "Otter-Video"
            master_print(f"The current model version is configured for {kind} with max_num_frames set to {self.max_num_frames}.")

        vision_encoder = CLIPVisionModel(config=config.vision_config)
        vision_encoder.output_tokens = True
        self.vision_encoder = vision_encoder
        self.vis_dim = 1024                                    # hard-coded in the reference (:798)
        self.perceiver = self._perceiver_cls(dim=self.vis_dim, max_num_frames=self.max_num_frames)
        self.lang_encoder.init_otter(media_token_id=self.media_token_id, vis_hidden_size=self.vis_dim,
                                     cross_attn_every_n_layers=self.cross_attn_every_n_layers,
                                     use_media_placement_augmentation=self.use_media_placement_augmentation)
        if "lora_config" in config.__dict__:
            self._wrap_lora(config)
        self.post_init()

    def _wrap_lora(self, config):
        """The reference's peft LoRA (:808-829), built by otter_b200.lora: peft's module and state-dict layout, with the
        adapters running on the otter_b200 decoder layers' kernels (peft's would be bypassed there)."""
        from .lora import wrap_lora
        arch = self.lang_encoder.__class__.__name__
        short = {"LlamaForCausalLM": "llama", "OPTForCausalLM": "opt", "GPTJForCausalLM": "gptj",
                 "GPTNeoXForCausalLM": "gpt_neox", "MPTForCausalLM": "mpt", "MosaicGPT": "mpt"}[
            config.text_config.architectures[0]]
        targets = {"llama": ["q_proj", "v_proj"], "opt": ["q_proj", "v_proj"], "gptj": ["q_proj", "v_proj"],
                   "gpt_neox": ["query_key_value"], "mpt": ["Wqkv"]}[short]
        lc = config.lora_config
        self.lang_encoder = wrap_lora(self.lang_encoder, r=lc["r"], lora_alpha=lc["lora_alpha"],
                                      lora_dropout=lc["lora_dropout"], target_modules=targets)
        self.lang_encoder.__class__.__name__ = f"{arch}LoRA"

    # ---- accessors (:833-849) ----
    def get_input_embeddings(self) -> nn.Module:
        return self.lang_encoder.get_input_embeddings()

    def set_input_embeddings(self, new_embeddings):
        self.lang_encoder.set_input_embeddings(new_embeddings)

    def get_output_embeddings(self) -> nn.Module:
        return self.lang_encoder.get_output_embeddings()

    def set_output_embeddings(self, new_embeddings):
        self.lang_encoder.set_output_embeddings(new_embeddings)

    def get_image_encoder(self) -> nn.Module:
        return self.vision_encoder

    def get_lang_encoder(self) -> nn.Module:
        return self.lang_encoder

    # ---- freeze policy (:851-915): everything frozen except perceiver, gated x-attn, embeddings ----
    def init_weights(self):
        flags = self.config.__dict__
        if not flags.get("train_full_model", False) is True:
            self.requires_grad_(False)
        if flags.get("train_vision_encoder", False) is True:
            master_print("Unfreeze vision encoder.")
            self.vision_encoder.requires_grad_(True)
        if flags.get("train_lang_encoder", False) is True:
            master_print("Unfreeze language decoder.")
            self.lang_encoder.requires_grad_(True)
        for name, param in self.lang_encoder.named_parameters():
            if "gated_cross_attn_layer" in name or ("lora_config" in flags and "lora" in name):
                param.requires_grad = True
        for name, param in self.named_parameters():
            if "perceiver" in name:
                param.requires_grad = True
        self.lang_encoder.get_input_embeddings().requires_grad_(True)
        if "LlamaForCausalLM" in self.lang_encoder.__class__.__name__:
            self.lang_encoder.lm_head.requires_grad_(True)
        total = 0
        for name, param in self.named_parameters():
            if param.requires_grad:
                total += param.numel()
                master_print(f"Parameter: {name}, Size: {param.numel() / 1e6:.6f} M")
        master_print(f"Total Trainable param: {total / 1e9:.6f} B")

    # ---- a-1 ----
    def _encode_vision_x(self, vision_x: torch.Tensor):
        """vision_x (B, T_img, F, C, H, W) -> condition every decoder layer on the resampled media tokens."""
        if self._assert_single_frame:
            assert vision_x.ndim == 6, "vision_x should be of shape (b, T_img, F, C, H, W)"
            assert vision_x.shape[2] == 1, "Only single frame supported"
        vis = encode_vision_x(self.vision_encoder, self.perceiver, vision_x)
        for layer in self.lang_encoder._get_decoder_layers():
            layer.condition_vis_x(vis)

    def forward(self, vision_x: torch.Tensor, lang_x: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                labels: Optional[torch.Tensor] = None, use_cached_vision_x: bool = False,
                clear_conditioned_layers: bool = True, past_key_values: Optional[List[torch.FloatTensor]] = None,
                use_cache: bool = False, **kwargs) -> CausalLMOutputWithPast:
        assert (vision_x is not None) or use_cached_vision_x, "Must provide either vision_x or use_cached_vision_x to True."
        if use_cached_vision_x:
            assert vision_x is None, "Expect vision_x to be None when use_cached_vision_x is True."
            assert self.lang_encoder.is_conditioned()
        else:
            self._encode_vision_x(vision_x=vision_x)
        output = self.lang_encoder(input_ids=lang_x, attention_mask=attention_mask, labels=labels,
                                   past_key_values=past_key_values, use_cache=use_cache, **kwargs)
        if clear_conditioned_layers:
            self.lang_encoder.clear_conditioned_layers()
        return output


class OtterModel(_OtterBase):
    """reference :539-736 (resizes LLaMA embeddings, :573-574)."""
    _resize_llama_embeddings = True


class OtterForConditionalGeneration(_OtterBase):
    """reference :739-1042."""

    @torch.no_grad()
    def generate(self, vision_x: torch.Tensor, lang_x: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                 **generate_kwargs):
        if hasattr(self, "_hf_hook"):
            from accelerate.hooks import AlignDevicesHook, add_hook_to_module
            add_hook_to_module(self.lang_encoder, AlignDevicesHook(execution_device=lang_x.device, io_same_device=True,
                                                                    place_submodules=False))
        num_beams = generate_kwargs.get("num_beams", 1)
        if num_beams > 1:
            vision_x = vision_x.repeat_interleave(num_beams, dim=0)
        self._encode_vision_x(vision_x=vision_x)
        output = self.lang_encoder.generate(input_ids=lang_x, attention_mask=attention_mask,
                                            eos_token_id=self.eoc_token_id, **generate_kwargs)
        self.lang_encoder.clear_conditioned_layers()
        return output
