"""H100-native mirror of the reference's `cambrian.model` package (the drop-in boundary, SURVEY.md §8b)."""
from .language_model.cambrian_llama import CambrianConfig, CambrianLlamaForCausalLM, CambrianLlamaModel  # noqa: F401
