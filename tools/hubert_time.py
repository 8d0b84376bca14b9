"""Time only the HuBERT leg of bench.py (same code path: run_hubert_gpu) and print its JSON."""
import sys, os, json, argparse
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from slamkit_b200 import _lib

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--dump-outputs", default=None, help="directory for the last batch's unit ids and frame counts (.npy)")
args = ap.parse_args()
lib = _lib.require_cuda()
out = bench.run_hubert_gpu(args, 0, 0, 1, lib, None)
print(json.dumps(out))
