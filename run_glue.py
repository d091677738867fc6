#!/usr/bin/env python
"""GLUE fine-tuning / evaluation / test prediction CLI for the classification tasks; implementation in
bert_pytorch_b200/finetune_glue.py."""
from bert_pytorch_b200.finetune_glue import main

if __name__ == "__main__":
    main()
