"""One encoder-half forward at the bench workload inside cudaProfilerStart/Stop, for ncu:

  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv \
      --log-file out/launches.csv python tools/profile_step.py
  ncu --profile-from-start off --set full --clock-control none --import-source on -k regex:msda_fwd \
      -o out/msda python tools/profile_step.py
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import salience_detr_b200 as pkg  # noqa: E402
from salience_detr_b200.synthetic import build_model, make_inputs  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", default="resnet50_800_1333_bs2")
ap.add_argument("--no-order", action="store_true")
ap.add_argument("--schedule", type=int, default=None)
ap.add_argument("--gemm", default="auto")
args = ap.parse_args()
if args.schedule is not None:
    import salience_detr_b200.salience_transformer as st
    st.MSDA_SCHEDULE = args.schedule
    st.SalienceTransformerEncoderLayer.forward_fast.__defaults__ = (None, args.schedule)

pkg.gemm.MODE = args.gemm
dev = torch.device("cuda:0")
model = build_model().to(dev)
feats, masks, pos = make_inputs(args.workload, seed=0, device=dev)
with torch.no_grad():
    plan = model.make_plan(masks)
    for _ in range(2):
        model.forward_encoder(feats, masks, pos, plan=plan, use_order=not args.no_order)
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    model.forward_encoder(feats, masks, pos, plan=plan, use_order=not args.no_order)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
print("launches", pkg.cabi.launch_count())
