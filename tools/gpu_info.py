"""The card a timing tool measured on, for the record it prints: every number the project states carries the GPU
model and its power limit."""
import subprocess

import torch


def gpu_info():
    """'name, power limit, max SM clock' of the visible GPU from one read-only nvidia-smi query; torch's device name
    and the query's error when it fails."""
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the name still comes from torch
        return "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(0), e)
