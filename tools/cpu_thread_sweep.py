"""Thread sweep of the CPU arm (oracle fp32 train step, B=1, S=128) on this host: justifies the thread count bench.py
uses for `cpu_baseline` / `--impl reference`.  Writes $MIDI_TOOLS_OUT/cpu_thread_sweep.txt."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.environ.get("MIDI_TOOLS_OUT", os.path.join(ROOT, "tools_out"))
code = ("import sys,os;sys.path.insert(0,%r);import bench;"
        "v,ms,c,s=bench.cpu_train_step_tokens_per_s('tv2o-medium',2,1);print('THREADS',c,'tok/s',round(v,1),'ms/step',round(ms,1))" % ROOT)
lines = [f"host cpu_count={os.cpu_count()}"]
for t in (8, 16, 32, 64, os.cpu_count() or 1):
    env = dict(os.environ, B200_CPU_THREADS=str(t))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600)
    out = [l for l in r.stdout.splitlines() if l.startswith("THREADS")]
    lines.append(out[0] if out else f"threads {t}: failed {r.stderr[-300:]}")
    print(lines[-1], flush=True)
os.makedirs(OUT_DIR, exist_ok=True)
open(os.path.join(OUT_DIR, "cpu_thread_sweep.txt"), "w").write("\n".join(lines) + "\n")
