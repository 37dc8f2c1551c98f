"""Dev aid: sweep the block schedule of the single-GPU look-ahead drivers.
  head: the remaining order above which the LLT's blocks are 512 wide (FAER_B200_LLT_HEAD; a value >= n leaves the
        256 / 128 schedule), LLT only;
  nb:   one block width (FAER_B200_NB) for the LLT and LU entry points.
usage: python tools/sweep_nb.py [head|nb] [sizes...]"""
import os
import subprocess
import sys

what = sys.argv[1] if len(sys.argv) > 1 and sys.argv[1] in ("head", "nb") else "nb"
sizes = [a for a in sys.argv[1:] if a not in ("head", "nb")] or ["16384"]
if what == "head":
    for head in ["16384", "12288", "10240", "8192", "7168"]:
        print(f"--- FAER_B200_LLT_HEAD={head}", flush=True)
        subprocess.run([sys.executable, "tools/time_factor.py", "llt"] + sizes, env=dict(os.environ, FAER_B200_LLT_HEAD=head))
    sys.exit(0)
for nb in ["512", "768", "1024", "1536", "2048"]:
    env = dict(os.environ, FAER_B200_NB=nb)
    print(f"--- FAER_B200_NB={nb}", flush=True)
    subprocess.run([sys.executable, "tools/time_factor.py", "all"] + sizes, env=env)
print("--- recursive drivers (FAER_B200_LOOKAHEAD_MIN_N=0)", flush=True)
subprocess.run([sys.executable, "tools/time_factor.py", "all"] + sizes, env=dict(os.environ, FAER_B200_LOOKAHEAD_MIN_N="0"))
