"""bert_pytorch_b200 -- a Hopper (sm_90a) native BERT pretraining / finetuning stack.

Layout
------
models/    BertConfig, the nn.Module model zoo (state-dict compatible with the
           reference, SURVEY.md 2.5.3) and the fused sm_90a execution engine
ops/       hand written CUDA kernels (csrc/) + their Python bindings
optim/     LAMB / Adam (fused multi-tensor kernels + pure-torch oracles),
           LR schedulers, gradient scaler
parallel/  communication backends (nccl / gloo / in-process fake / fused
           peer-memory) and the data-parallel engine
data/      native HDF5 reader/writer, sharded dataset, resumable sampler,
           dynamic masking, SQuAD / NER featurisers, tokenisation
kfac/      K-FAC preconditioner
utils/     logging sinks, checkpointing, device timing, distributed helpers
"""

__version__ = "0.1.0"

from .config import BertConfig  # noqa: F401
