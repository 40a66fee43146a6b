"""Times the fused loss kernel at GraphCast 0.25 degree / 37 levels (721 x 1440 grid, 227 output
channels) against the plain output unpack, with CUDA events after warm-ups:

  unpack       gcb_unpack_grid_outputs (predictions only; what GraphCast.__call__ runs)
  loss         gcb_output_loss without planes_out (GraphCast.loss / InputsAndResiduals.loss)
  loss+preds   gcb_output_loss with planes_out (loss_and_predictions)

all with the residual normalisation of InputsAndResiduals (scale, offset and an add plane for every
channel, the worst case).  Bytes are the algorithmic HBM traffic computed from the shapes; the rate
is compared with the H100 SXM data-sheet bandwidth of 3.35 TB/s.  Prints the card, its power limit
and SM clock limit next to the numbers.  Needs a GPU; there is no CPU mode.

  python tools/time_loss.py [--reps 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from graphcast_b200 import _native  # noqa: E402

PEAK_BW = 3.35e12


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=50)
  ap.add_argument("--warmup", type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("time_loss.py needs a CUDA device")
  lib = _native.lib()
  dev = torch.device("cuda:0")
  n_lat, n_lon, n_out, ld = 721, 1440, 227, 256
  n = n_lat * n_lon
  g = torch.Generator(device=dev).manual_seed(0)
  y = torch.randn(n, ld, device=dev, generator=g)
  targets = torch.randn(n_out, n, device=dev, generator=g)
  add = torch.randn(n_out, n, device=dev, generator=g)
  scale = torch.rand(n_out, device=dev, generator=g) + 0.5
  offset = torch.zeros(n_out, device=dev)
  idx = torch.arange(n_out, dtype=torch.int32, device=dev)
  w = torch.rand(n_lat, device=dev, generator=g)
  planes = torch.empty(n_out, n, device=dev)
  sums = torch.empty(n_out, dtype=torch.float64, device=dev)
  nbytes = lib.gcb_output_loss_workspace_bytes(n_out)
  ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
  st = torch.cuda.current_stream().cuda_stream

  def unpack():
    _native.check(lib.gcb_unpack_grid_outputs(y.data_ptr(), ld, n_out, n, scale.data_ptr(),
                                              offset.data_ptr(), add.data_ptr(), idx.data_ptr(),
                                              planes.data_ptr(), st), "unpack")

  def loss(with_planes):
    _native.check(lib.gcb_output_loss(y.data_ptr(), ld, n_out, n_lat, n_lon, scale.data_ptr(),
                                      offset.data_ptr(), add.data_ptr(), idx.data_ptr(),
                                      targets.data_ptr(), w.data_ptr(),
                                      planes.data_ptr() if with_planes else None, ws.data_ptr(),
                                      nbytes, sums.data_ptr(), st), "loss")

  elem = 4.0 * n * n_out
  cases = [("unpack", unpack, 3 * elem),                       # y, add read; predictions written
           ("loss", lambda: loss(False), 3 * elem),            # y, add, targets read
           ("loss+preds", lambda: loss(True), 4 * elem)]       # ... and predictions written
  results = {}
  for _ in range(2):                                           # alternate the cases twice
    for name, fn, bytes_ in cases:
      for _ in range(args.warmup):
        fn()
      beg, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      torch.cuda.synchronize()
      beg.record()
      for _ in range(args.reps):
        fn()
      end.record()
      end.synchronize()
      ms = beg.elapsed_time(end) / args.reps
      results.setdefault(name, []).append(ms)
  try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True,
                          check=True).stdout.strip()
  except (OSError, subprocess.CalledProcessError):
    card = torch.cuda.get_device_name(0)
  print(f"card: {card}")
  out = {"card": card, "grid": [n_lat, n_lon], "n_out": n_out}
  for name, _, bytes_ in cases:
    ms = min(results[name])
    print(f"{name:11s} {ms:7.3f} ms  {bytes_ / 1e9:5.2f} GB  {bytes_ / ms / 1e6:6.0f} GB/s  "
          f"{100 * bytes_ / ms / 1e-3 / PEAK_BW:4.1f} % of 3.35 TB/s   (runs: "
          + ", ".join(f"{m:.3f}" for m in results[name]) + ")")
    out[name] = {"ms": ms, "gb": bytes_ / 1e9, "runs_ms": results[name]}
  print(json.dumps(out))


if __name__ == "__main__":
  main()
