# compute-sanitizer on the final kernels: memcheck (humanoid3d, dog3d, target_amp task variant, plain and gated policy networks, discriminator reward), racecheck (humanoid3d)
set -x
timeout 900 compute-sanitizer --tool memcheck --print-limit 5 python tools/sanitize_run.py 2>&1 | tail -6
timeout 900 compute-sanitizer --tool memcheck --print-limit 5 python tools/sanitize_run.py args/train_dog3d_trot_args.txt 2>&1 | tail -4
timeout 900 compute-sanitizer --tool memcheck --print-limit 5 python tools/mlp_time.py 2>&1 | tail -4
timeout 900 compute-sanitizer --tool racecheck --print-limit 5 python tools/sanitize_run.py 2>&1 | tail -8
