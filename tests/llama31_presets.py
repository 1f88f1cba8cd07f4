"""Oracle configurations of the engine's Llama-3.1 presets (csrc/model_config.cc model_preset) — TEST SIDE.

Each is the oracle preset of the same shapes and seeded weights (tiny, llama-3-8b-l2, llama-3-8b) with Llama-3.1's
"llama3" RoPE scaling (factor 8, low 1, high 4, original 8192) and 131072-token window.
tests/test_long_context_cpu.py checks that the engine describes the same models.
"""
import dataclasses

from oracle.llama_oracle import PRESETS

BASE = {"tiny-3.1": "tiny", "llama-3.1-8b-l2": "llama-3-8b-l2", "llama-3.1-8b": "llama-3-8b"}
LLAMA31 = {name: dataclasses.replace(PRESETS[base], name=name, max_pos=131072, rope_scaling=(8.0, 1.0, 4.0, 8192))
           for name, base in BASE.items()}
