"""The configuration of the downstream-script runs (tests/golden/make_golden_finetune.py produces the goldens with the
reference's own modules on CPU, tests/test_gpu_zz_finetune_scripts.py runs the same scripts against this package on the
GPU): mn04_as from its release file (so "Dropping last layer" runs), two epochs over 24 one-second synthetic clips,
no roll / waveform mixing / gain augmentation (the synthetic stand-ins have none)."""
ENV = {"EAT_SYNTH_CLIP_SECONDS": "1", "EAT_SYNTH_TRAIN_CLIPS": "24", "EAT_SYNTH_TEST_CLIPS": "20"}
COMMON = ["--pretrained", "--model_name", "mn04_as", "--batch_size", "8", "--num_workers", "0", "--n_epochs", "2",
          "--no_roll", "--no_wavmix", "--gain_augment", "0", "--warm_up_len", "1", "--ramp_down_start", "1",
          "--ramp_down_len", "2", "--last_lr_value", "0.1", "--lr", "2e-4"]
# golden name -> (script, extra arguments)
RUNS = {"esc50": ("ex_esc50.py", []),
        "dcase20": ("ex_dcase20.py", []),
        "dcase20_mixstyle": ("ex_dcase20.py", ["--mixstyle_p", "1"]),
        "fsd50k": ("ex_fsd50k.py", ["--train", "--variable_eval_length"]),
        "openmic": ("ex_openmic.py", ["--train"])}
# one golden file per task: tests/golden/script_<task>.json holds every run of that task
TASK = {"esc50": "esc50", "dcase20": "dcase20", "dcase20_mixstyle": "dcase20", "fsd50k": "fsd50k", "openmic": "openmic"}
