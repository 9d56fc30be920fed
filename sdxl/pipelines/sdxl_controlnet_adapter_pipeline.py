"""/root/reference/sdxl/pipelines/sdxl_controlnet_adapter_pipeline.py: the pipeline class inference.py imports (:363),
backed by the H100 denoising loop (pipeline body :1279-1404)."""
from ctrl_adapter_b200.pipeline_sdxl import SDXLControlNetAdapterLoop  # noqa: F401
from ctrl_adapter_b200.pipelines import SDXLControlNetAdapterPipeline, StableDiffusionXLPipelineOutput  # noqa: F401
