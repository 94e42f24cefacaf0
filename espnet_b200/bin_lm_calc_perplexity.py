"""Command line of espnet2/bin/lm_calc_perplexity.py on the CUDA path: ``python -m espnet_b200.bin_lm_calc_perplexity --output_dir DIR
--data_path_and_name_and_type data/test/text,text,text --train_config lm/config.yaml --model_file lm/valid.loss.best.pth``.

Same option names and defaults as the reference (lm_calc_perplexity.py:134-203), except ``--ngpu``, which defaults to 1 (there is no CPU
path) and ``--dtype``, which accepts float32 only."""
import argparse
import sys

from .lm_calc_perplexity import calc_perplexity


def _none_or(conv):
    return lambda v: None if str(v).strip().lower() in ("none", "null", "nil", "") else conv(v)


def _str2bool(v):
    s = str(v).strip().lower()
    if s in ("y", "yes", "t", "true", "on", "1"):
        return True
    if s in ("n", "no", "f", "false", "off", "0"):
        return False
    raise argparse.ArgumentTypeError(f"invalid truth value {v!r}")


def _triple(v):
    v = v.strip()
    if v.startswith("(") and v.endswith(")"):
        v = v[1:-1]
    a, b, c = v.split(",")
    return a.strip(), b.strip(), c.strip()


def get_parser():
    p = argparse.ArgumentParser(description="Calc perplexity (espnet_b200)", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument("--log_level", type=lambda x: x.upper(), default="INFO", choices=("CRITICAL", "ERROR", "WARNING", "INFO", "DEBUG", "NOTSET"))
    p.add_argument("--output_dir", type=str, required=True)
    p.add_argument("--ngpu", type=int, default=1, help="The number of gpus (the CUDA path needs at least one)")
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--dtype", default="float32", choices=["float32"])
    p.add_argument("--num_workers", type=int, default=1)
    p.add_argument("--batch_size", type=int, default=1)
    p.add_argument("--log_base", type=_none_or(float), default=None, help="The base of logarithm for Perplexity (None: e)")
    g = p.add_argument_group("Input data related")
    g.add_argument("--data_path_and_name_and_type", type=_triple, required=True, action="append")
    g.add_argument("--key_file", type=_none_or(str))
    g.add_argument("--allow_variable_data_keys", type=_str2bool, default=False)
    g = p.add_argument_group("The model configuration related")
    g.add_argument("--train_config", type=str)
    g.add_argument("--model_file", type=str)
    return p


def main(cmd=None):
    print(" ".join(sys.argv), file=sys.stderr)
    args = vars(get_parser().parse_args(cmd))
    args.pop("config", None)
    calc_perplexity(**args)


if __name__ == "__main__":
    main()
