"""/root/reference/svd/pipelines/svd_controlnet_adapter_pipeline.py: the pipeline class inference.py imports (:358),
backed by the H100 denoising loop (pipeline body :640-787)."""
from ctrl_adapter_b200.pipeline_svd import SVDControlNetAdapterLoop  # noqa: F401
from ctrl_adapter_b200.pipelines import SVDControlNetAdapterPipeline, StableVideoDiffusionPipelineOutput  # noqa: F401
