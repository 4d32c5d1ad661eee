"""Runs the bench workload once per environment-variable setting (tuning hooks such as
MSD_ATTN_TAIL / MSD_FUSED_NORM) in separate processes and prints one summary line each."""
import json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
  settings = sys.argv[1:] or ['']
  for s in settings:
    env = dict(os.environ)
    for kv in filter(None, s.split(',')):
      k, v = kv.split('=')
      env[k] = v
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--steps', '2', '--warmup', '1',
                          '--no-cpu-baseline', '--no-song', '--diffusion-steps', '300', '--segments',
                          env.get('SWEEP_SEGMENTS', '8')], env=env, cwd=ROOT,
                         capture_output=True, text=True, timeout=600)
    line = [l for l in out.stdout.splitlines() if l.startswith('{')]
    if not line:
      print(f'{s or "default"}: FAILED rc={out.returncode} {out.stderr[-400:]}', flush=True)
      continue
    j = json.loads(line[-1])
    print(f'{s or "default"}: value={j["value"]:.1f} e2e={j["e2e"]["value"]:.1f} '
          f'classes={j.get("kernel_classes_ms_per_diffusion_step")}', flush=True)


if __name__ == '__main__':
  main()
