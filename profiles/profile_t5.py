"""One eager flan-T5-XL encoder forward (5 prompts x 100 tokens) between cudaProfilerStart/Stop, for
  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file launches_t5.csv python profiles/profile_t5.py"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ezaudio_b200 import synth, weights  # noqa: E402
from ezaudio_b200.t5 import T5EncoderModel  # noqa: E402

cfg = dict(synth.T5_XL, num_layers=int(os.environ.get("T5_LAYERS", 4)))   # the layers are identical: a few are enough for the launch list
sd = weights.synthetic_state_dict(weights.t5_param_shapes(cfg), 15)
t5 = T5EncoderModel(cfg, max_batch=5, max_len=100).load_state_dict(sd)
t5.use_graphs = False
ids, mask = synth.synth_tokens(5, 100, cfg["vocab_size"])
ids, mask = ids.cuda(), mask.cuda()
for _ in range(2):
    t5(input_ids=ids, attention_mask=mask)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStart()
t5(input_ids=ids, attention_mask=mask)
torch.cuda.synchronize()
torch.cuda.cudart().cudaProfilerStop()
