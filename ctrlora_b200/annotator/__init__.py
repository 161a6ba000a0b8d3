"""Condition-image annotators on the sm_90a kernels: line art (`ctrlora_b200.annotator.lineart`), HED
(`ctrlora_b200.annotator.hed`) and HED-sketch (`ctrlora_b200.annotator.hedsketch`).  The reference's other detectors
stay its own `annotator` package."""
