"""Condition-image annotators on the sm_90a kernels: line art (`ctrlora_b200.annotator.lineart`), anime line art
(`ctrlora_b200.annotator.lineart_anime`), HED (`ctrlora_b200.annotator.hed`), HED-sketch (`ctrlora_b200.annotator.hedsketch`), OpenPose bodies
(`ctrlora_b200.annotator.openpose`), MiDaS depth and normals (`ctrlora_b200.annotator.midas`), UniFormer
segmentation (`ctrlora_b200.annotator.uniformer`) and M-LSD straight lines (`ctrlora_b200.annotator.mlsd`).  The
reference's other detectors stay its own `annotator` package."""
