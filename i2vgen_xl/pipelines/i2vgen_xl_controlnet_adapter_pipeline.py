"""/root/reference/i2vgen_xl/pipelines/i2vgen_xl_controlnet_adapter_pipeline.py: the pipeline class inference.py imports
(:351), backed by the H100 denoising loop (pipeline body :902-1118)."""
from ctrl_adapter_b200.pipeline_i2vgen import I2VGenXLControlNetAdapterLoop  # noqa: F401
from ctrl_adapter_b200.pipelines import I2VGenXLControlNetAdapterPipeline, I2VGenXLPipelineOutput  # noqa: F401
