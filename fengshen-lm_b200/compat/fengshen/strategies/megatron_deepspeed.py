"""`fengshen.strategies.megatron_deepspeed.DeepSpeedStrategy` — constructor signature of
fengshen/strategies/megatron_deepspeed.py:55-104 (positional pipe/tensor sizes + mpu_seed, then the ZeRO knobs), config
discovery through $PL_DEEPSPEED_CONFIG_PATH (:53) and the `activation_checkpointing` assertion (:326-327). The engine it
configures is fsb200.engine.ZeroEngine instead of deepspeed.initialize (:302-320)."""
from pytorch_lightning.strategies.deepspeed import DeepSpeedStrategy as OriginDeepSpeedStrategy

from fengshen.models.megatron import mpu, fused_kernels


class DeepSpeedStrategy(OriginDeepSpeedStrategy):
    strategy_name = "megatron_deepspeed"
    DEEPSPEED_ENV_VAR = "PL_DEEPSPEED_CONFIG_PATH"

    def __init__(self, pipe_model_parallel_size, tensor_model_parallel_size, mpu_seed, accelerator=None,
                 zero_optimization=True, stage=2, **kwargs):
        if pipe_model_parallel_size != 1:
            raise NotImplementedError("fsb200: pipe_model_parallel_size must be 1 (pipeline parallelism is outside the hot path)")
        super().__init__(accelerator=accelerator, zero_optimization=zero_optimization, stage=stage, **kwargs)
        self.pipe_model_parallel_size = pipe_model_parallel_size
        self.tensor_model_parallel_size = tensor_model_parallel_size
        self.mpu_seed = mpu_seed

    def setup_mpu(self, trainer):
        """megatron_deepspeed.py:339-369 at PP = 1: load the kernels, build the tensor- / data-parallel groups, seed."""
        fused_kernels.load_fused_kernels()
        mpu.initialize_model_parallel(self.tensor_model_parallel_size, self.pipe_model_parallel_size)
        # The `activation_checkpointing` block is accepted and ignored. In DeepSpeed it only configures
        # deepspeed.checkpointing.checkpoint, which the reference model never calls (SURVEY §2.4), so honouring it would change
        # the speed and memory of unmodified recipe runs. Recompute is the model's own switch: gradient_checkpointing_enable().
        if "activation_checkpointing" in self.config:
            pass
        import torch
        torch.manual_seed(self.mpu_seed)
