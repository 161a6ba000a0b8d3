"""Condition-image annotators on the sm_90a kernels.  Only line art (`ctrlora_b200.annotator.lineart`) is implemented;
the reference's other detectors stay its own `annotator` package."""
