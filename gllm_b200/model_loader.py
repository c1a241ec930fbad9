"""Config + weights loading (reference: gllm/model_loader.py:34-181).

Checkpoint format = stock HuggingFace directories (`config.json`, `generation_config.json`,
tokenizer files, `*.safetensors` or `*.bin`). `load_format="dummy"` builds random weights;
`model_path="preset:<name>"` uses a built-in config (no files needed).
"""
from __future__ import annotations

import json
import os
from typing import Optional

import torch

from gllm_b200.models import registry
from gllm_b200.models.presets import PRESETS
from gllm_b200.models.weight_utils import CheckpointReader
from gllm_b200.utils.logging import logger


class ModelLoader:
    def __init__(self, model_path, load_format: str = "auto", quantization: Optional[str] = None):
        self.model_path = model_path
        self.load_format = load_format
        self.config = self.load_config(model_path)
        if quantization is not None:     # validated with the checkpoint's own config by registry.build_model
            self.config[registry.QUANTIZATION_KEY] = quantization
        self.generation_config = self.load_generation_config(model_path)
        self.architecture = self.config["architectures"][0]
        self.use_mla = self.architecture in ("DeepseekV2ForCausalLM", "DeepseekV3ForCausalLM") and \
            self.config.get("kv_lora_rank") is not None
        self.config["use_mla"] = self.use_mla
        self.use_mm = self.architecture in ("Qwen2_5_VLForConditionalGeneration",
                                            "Qwen3VLForConditionalGeneration",
                                            "Qwen3VLMoeForConditionalGeneration")

    @staticmethod
    def load_config(model_path) -> registry.HFConfig:
        if isinstance(model_path, dict):
            return registry.HFConfig(dict(model_path))
        if isinstance(model_path, str) and model_path.startswith("preset:"):
            name = model_path.split(":", 1)[1]
            if name not in PRESETS:
                raise ValueError(f"unknown preset {name}; available: {sorted(PRESETS)}")
            return registry.HFConfig(dict(PRESETS[name]))
        cfg_path = os.path.join(model_path, "config.json")
        if not os.path.exists(cfg_path):
            raise FileNotFoundError(
                f"{cfg_path} not found (model_path must be a local HuggingFace directory or preset:<name>)")
        with open(cfg_path) as f:
            cfg = registry.HFConfig(json.load(f))
        # VL checkpoints nest the language model config
        if "text_config" in cfg and "hidden_size" not in cfg:
            merged = dict(cfg["text_config"])
            merged.update({k: v for k, v in cfg.items() if k != "text_config"})
            cfg = registry.HFConfig(merged)
        return cfg

    @staticmethod
    def load_generation_config(model_path) -> dict:
        if isinstance(model_path, str) and not model_path.startswith("preset:"):
            p = os.path.join(model_path, "generation_config.json")
            if os.path.exists(p):
                with open(p) as f:
                    return json.load(f)
        return {}

    def eos_token_ids(self):
        eos = self.generation_config.get("eos_token_id", self.config.get("eos_token_id"))
        if eos is None:
            return []
        return list(eos) if isinstance(eos, (list, tuple)) else [eos]

    def load_model(self, device, progress=None):
        model = registry.build_model(self.config, device)
        if self.load_format == "dummy" or isinstance(self.model_path, dict) or \
                (isinstance(self.model_path, str) and self.model_path.startswith("preset:")):
            model.init_dummy()
        else:
            reader = CheckpointReader(self.model_path)
            model.load_weights(reader, progress)
        if hasattr(model, "process_weights"):
            model.process_weights()
        n_bytes = sum(p.numel() * p.element_size() for p in model.parameters())
        logger.info("model %s: %.2f GB of weights on this rank", self.architecture, n_bytes / 2 ** 30)
        return model
