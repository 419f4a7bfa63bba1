"""lora_b200 -- Hopper-native (sm_90a) LoRA fine-tuning hot path behind the API of
cloneofsimo/lora (`lora_diffusion`). See INTEGRATION.md."""
from .lora import *  # noqa: F401,F403
from .lora import (_find_children, _find_modules, _find_modules_v2, _text_lora_path,  # noqa: F401
                   _ti_lora_path)

from .modules import get_fp32_mode, set_fp32_mode  # noqa: F401,E402
from .grouping import get_grouping, link_sites, set_grouping  # noqa: F401,E402
# lora_diffusion/__init__.py:5 re-exports lora_manager's names at package level
from .join import DummySafeTensorObject, LoRAManager, lora_join  # noqa: F401,E402

__version__ = "0.1.0"
