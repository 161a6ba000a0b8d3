"""Host-side mirror of the reference's module contract (SURVEY.md §8b).

`ctrlora_b200/dropin` is a directory of top-level packages named like the reference's (`cldm`, `ldm`): put it first
on sys.path (see `activate()`) and `cldm.model.create_model`, the YAML `target:` strings, `cldm.lora`,
`cldm.ddim_hacked.DDIMSampler`, `ldm.modules.attention`, `ldm.modules.diffusionmodules.openaimodel` resolve to the
H100-native implementation.  INTEGRATION.md shows the file-level overlay onto a reference checkout.
"""
import os
import sys

DROPIN_ROOT = os.path.dirname(os.path.abspath(__file__))


def activate():
    """Make `import cldm` / `import ldm` resolve to this implementation (idempotent)."""
    if DROPIN_ROOT not in sys.path:
        sys.path.insert(0, DROPIN_ROOT)
    for name in list(sys.modules):
        if name in ("cldm", "ldm") or name.startswith(("cldm.", "ldm.")):
            mod = sys.modules[name]
            f = getattr(mod, "__file__", "") or ""
            if not f.startswith(DROPIN_ROOT):
                del sys.modules[name]  # a foreign (reference) copy was imported earlier: drop it
    return DROPIN_ROOT
