"""
Command line of badread_b200: `python -m badread_b200 simulate ...` with the flags, defaults and validation
messages of `badread simulate` (/root/reference/badread/__main__.py:83-147, 239-336). Additive flags: --gpus,
--batch_reads. `error_model` and `qscore_model` take the reference's arguments, and their --alignment may also be SAM or
BAM (then --reads is optional). `plot` takes the reference's arguments, computes the window series on the GPU and
does not draw: --no_plot prints what the reference prints, and the additive --windows FILE writes the series as a
table (its --alignment may also be SAM or BAM).

Derived from Badread (Copyright 2018 Ryan Wick, rrwick@gmail.com, https://github.com/rrwick/Badread), which is free
software under the GNU General Public License version 3 or later; this file mirrors the named parts of the
reference's interface and is distributed under the same licence (see LICENSE and NOTICE at the repository root).
"""
import argparse
import pathlib
import sys

from . import settings
from .misc import str_is_dna_sequence, str_is_int
from .version import __version__


def main(output=sys.stderr):
    args = parse_args(sys.argv[1:])
    if args.subparser_name == 'simulate':
        check_simulate_args(args)
        from .simulate import simulate
        simulate(args, output=output)
    elif args.subparser_name == 'error_model':
        from .model_builders import make_error_model
        make_error_model(args, output=output)
    elif args.subparser_name == 'qscore_model':
        from .model_builders import make_qscore_model
        make_qscore_model(args, output=output)
    elif args.subparser_name == 'plot':
        if not args.no_plot and args.windows is None:
            sys.exit('Error: badread_b200 does not draw plots: write the window series with --windows FILE, or use '
                     '--no_plot')
        from .plot import plot_window_identity
        plot_window_identity(args, output=sys.stdout)
    else:
        sys.exit(f'Error: the {args.subparser_name} command is not part of badread_b200 (use Badread itself)')


def parse_args(args):
    parser = argparse.ArgumentParser(prog='badread', description='Badread: a long read simulator that can imitate '
                                     'many types of read problems (GPU build of the simulate command)')
    subparsers = parser.add_subparsers(title='Commands', dest='subparser_name')
    simulate_subparser(subparsers)
    model_subparser(subparsers, 'error_model', 'Build a Badread error model', 7)
    model_subparser(subparsers, 'qscore_model', 'Build a Badread qscore model', 9)
    plot_subparser(subparsers)
    parser.add_argument('--version', action='version', version='Badread v' + __version__)
    if len(args) == 0:
        parser.print_help(file=sys.stderr)
        sys.exit(1)
    parsed = parser.parse_args(args)
    if parsed.subparser_name in ('error_model', 'qscore_model') and parsed.reads is None:
        from .model_builders import alignment_format
        if alignment_format(parsed.alignment) == 'paf':   # (SAM and BAM records can carry the reads)
            subparsers.choices[parsed.subparser_name].error('the following arguments are required: --reads')
    return parsed


def model_subparser(subparsers, name, description, default_k):
    """The arguments of `badread error_model` / `badread qscore_model` (__main__.py:150-208 of the reference); --alignment
    may also be SAM or BAM, and then --reads may be left out."""
    group = subparsers.add_parser(name, description=description)
    required = group.add_argument_group('Required arguments')
    required.add_argument('--reference', type=str, required=True, help='Reference FASTA file')
    required.add_argument('--reads', type=str,
                          help='FASTQ of real reads (optional for a SAM or BAM alignment: the reads are then taken from '
                               'its records)')
    required.add_argument('--alignment', type=str, required=True,
                          help='Alignment of reads to the reference: PAF with cg:Z: and AS:i: tags, or SAM / BAM with '
                               'AS:i: tags (told apart by content)')
    optional = group.add_argument_group('Optional arguments')
    what = 'error' if name == 'error_model' else 'qscore'
    optional.add_argument('--k_size', type=int, default=default_k,
                          help=f'{what.capitalize()} model k-mer size' + (' (must be odd)' if what == 'qscore' else ''))
    optional.add_argument('--max_alignments', type=int,
                          help=f'Only use this many alignments when generating {what} model (default: use all alignments)')
    if name == 'error_model':
        optional.add_argument('--max_alt', type=int, default=25, help='Only save up to this many alternatives to each k-mer')
    else:
        optional.add_argument('--max_del', type=int, default=6,
                              help='Deletion runs longer than this will be collapsed to reduce the number of possible alignments')
        optional.add_argument('--min_occur', type=int, default=100,
                              help='CIGARs which occur less than this many times will not be included in the model')
        optional.add_argument('--max_output', type=int, default=10000,
                              help='The outputted model will be limited to this many lines')
    group.add_argument('--version', action='version', version='Badread v' + __version__)


def positive_int(text):
    value = int(text)
    if value < 1:
        raise argparse.ArgumentTypeError(f'must be at least 1: {text}')
    return value


def plot_subparser(subparsers):
    """The arguments of `badread plot` (__main__.py:212-236 of the reference) and --windows; --window must be at least 1."""
    group = subparsers.add_parser('plot', description='View read identities over a sliding window')
    required = group.add_argument_group('Required arguments')
    required.add_argument('--reference', type=str, required=True, help='Reference FASTA file')
    required.add_argument('--reads', type=str, required=True, help='FASTQ of real reads')
    required.add_argument('--alignment', type=str, required=True,
                          help='Alignment of reads to the reference: PAF with cg:Z: and AS:i: tags, or SAM / BAM with '
                               'AS:i: tags (told apart by content)')
    optional = group.add_argument_group('Optional arguments')
    optional.add_argument('--window', type=positive_int, default=100, help='Window size in bp')
    optional.add_argument('--qual', action='store_true', help='Include qscores in plot (default: only show identity)')
    optional.add_argument('--no_plot', action='store_true', help='Do not display plots (for testing purposes)')
    optional.add_argument('--windows', type=str,
                          help='Write the window series to this file as tab-separated lines: read name, position, '
                               'identity and, with --qual, mean qscore (BGZF when the name ends in .gz)')
    group.add_argument('--version', action='version', version='Badread v' + __version__)


def simulate_subparser(subparsers):
    group = subparsers.add_parser('simulate', description='Generate fake long reads')
    required_args = group.add_argument_group('Required arguments')
    required_args.add_argument('--reference', type=str, required=True, help='Reference FASTA file (can be gzipped)')
    required_args.add_argument('--quantity', type=str, required=True,
                               help='Either an absolute value (e.g. 250M) or a relative depth (e.g. 25x)')
    sim_args = group.add_argument_group('Simulation parameters')
    sim_args.add_argument('--length', type=str, default='15000,13000',
                          help='Fragment length distribution (mean and stdev, default: %(default)s)')
    sim_args.add_argument('--identity', type=str, default='95,99,2.5',
                          help='Sequencing identity distribution (mean,max,stdev for beta distribution or '
                               'mean,stdev for normal qscore distribution, default: %(default)s)')
    sim_args.add_argument('--error_model', type=str, default='nanopore2023',
                          help='Can be "nanopore2018", "nanopore2020", "nanopore2023", "pacbio2016", '
                               '"pacbio2021", "random" or a model filename')
    sim_args.add_argument('--qscore_model', type=str, default='nanopore2023',
                          help='Can be "nanopore2018", "nanopore2020", "nanopore2023", "pacbio2016", '
                               '"pacbio2021", "random", "ideal" or a model filename')
    sim_args.add_argument('--seed', type=int,
                          help='Random number generator seed for deterministic output (default: different '
                               'output each time)')
    adapter_args = group.add_argument_group('Adapters')
    adapter_args.add_argument('--start_adapter', type=str, default='90,60',
                              help='Adapter parameters for read starts (rate and amount, default: %(default)s)')
    adapter_args.add_argument('--end_adapter', type=str, default='50,20',
                              help='Adapter parameters for read ends (rate and amount, default: %(default)s)')
    adapter_args.add_argument('--start_adapter_seq', type=str, default='AATGTACTTCGTTCAGTTACGTATTGCT',
                              help='Adapter sequence for read starts')
    adapter_args.add_argument('--end_adapter_seq', type=str, default='GCAATACGTAACTGAACGAAGT',
                              help='Adapter sequence for read ends')
    problem_args = group.add_argument_group('Problems')
    problem_args.add_argument('--junk_reads', type=float, default=1,
                              help='This percentage of reads will be low-complexity junk')
    problem_args.add_argument('--random_reads', type=float, default=1,
                              help='This percentage of reads will be random sequence')
    problem_args.add_argument('--chimeras', type=float, default=1,
                              help='Percentage at which separate fragments join together')
    problem_args.add_argument('--glitches', type=str, default='10000,25,25',
                              help='Read glitch parameters (rate, size and skip, default: %(default)s)')
    problem_args.add_argument('--small_plasmid_bias', action='store_true',
                              help='If set, then small circular plasmids are lost when the fragment length is '
                                   'too high (default: small plasmids are included regardless of fragment length)')
    b200_args = group.add_argument_group('GPU')
    b200_args.add_argument('--gpus', type=int, default=1, help='GPUs to shard reads over (default: %(default)s)')
    b200_args.add_argument('--batch_reads', type=int, default=16384,
                           help='Reads per GPU per batch (default: %(default)s)')
    b200_args.add_argument('--gzip', action='store_true',
                           help='Write the FASTQ as BGZF (gzip-compatible), compressed on the GPUs')
    b200_args.add_argument('--bam', action='store_true',
                           help='Write unaligned BAM instead of FASTQ, built and compressed on the GPUs')
    group.add_argument('--version', action='version', version='Badread v' + __version__)


def check_simulate_args(args):
    """__main__.py:239-313, same messages."""
    if not pathlib.Path(args.reference).is_file():
        sys.exit(f'Error: {args.reference} is not a file')
    error_model_names = ['random', 'nanopore2018', 'nanopore2020', 'nanopore2023', 'pacbio2016', 'pacbio2021']
    if args.error_model.lower() not in error_model_names and not pathlib.Path(args.error_model).is_file():
        sys.exit(f'Error: {args.error_model} is not a file\n'
                 f'  --error_model must be from {error_model_names} or a filename')
    qscore_model_names = ['random', 'ideal', 'nanopore2018', 'nanopore2020', 'nanopore2023', 'pacbio2016',
                          'pacbio2021']
    if args.qscore_model.lower() not in qscore_model_names and not pathlib.Path(args.qscore_model).is_file():
        sys.exit(f'Error: {args.qscore_model} is not a file\n'
                 f'  --qscore_model must be from {qscore_model_names} or a filename')
    if args.chimeras > 50:
        sys.exit('Error: --chimeras cannot be greater than 50')
    if args.junk_reads > 100:
        sys.exit('Error: --junk_reads cannot be greater than 100')
    if args.random_reads > 100:
        sys.exit('Error: --random_reads cannot be greater than 100')
    if args.junk_reads + args.random_reads > 100:
        sys.exit('Error: --junk_reads and --random_reads cannot sum to more than 100')
    try:
        length_parameters = [float(x) for x in args.length.split(',')]
        args.mean_frag_length = length_parameters[0]
        args.frag_length_stdev = length_parameters[1]
    except (ValueError, IndexError):
        sys.exit('Error: could not parse --length values')
    if args.mean_frag_length <= settings.MIN_MEAN_READ_LENGTH:
        sys.exit(f'Error: mean read length must be at least {settings.MIN_MEAN_READ_LENGTH}')
    if args.frag_length_stdev < 0:
        sys.exit('Error: read length stdev cannot be negative')
    try:
        identity_parameters = [float(x) for x in args.identity.split(',')]
        if len(identity_parameters) == 2:
            args.mean_identity = identity_parameters[0]
            args.max_identity = None
            args.identity_stdev = identity_parameters[1]
            check_qscore_identities(args)
        elif len(identity_parameters) == 3:
            args.mean_identity = identity_parameters[0]
            args.max_identity = identity_parameters[1]
            args.identity_stdev = identity_parameters[2]
            check_beta_identities(args)
        else:
            sys.exit('Error: could not parse --identity values')
    except (ValueError, IndexError):
        sys.exit('Error: could not parse --identity values')
    try:
        glitch_parameters = [float(x) for x in args.glitches.split(',')]
        args.glitch_rate = glitch_parameters[0]
        args.glitch_size = glitch_parameters[1]
        args.glitch_skip = glitch_parameters[2]
    except (ValueError, IndexError):
        sys.exit('Error: could not parse --glitches values')
    if args.glitch_rate < 0 or args.glitch_size < 0 or args.glitch_skip < 0:
        sys.exit('Error: --glitches must contain non-negative values')
    if args.start_adapter_seq != '':
        if not str_is_int(args.start_adapter_seq):
            args.start_adapter_seq = args.start_adapter_seq.upper()
            if not str_is_dna_sequence(args.start_adapter_seq):
                sys.exit('Error: --start_adapter_seq must be a DNA sequence or a number')
    if args.end_adapter_seq != '':
        if not str_is_int(args.end_adapter_seq):
            args.end_adapter_seq = args.end_adapter_seq.upper()
            if not str_is_dna_sequence(args.end_adapter_seq):
                sys.exit('Error: --end_adapter_seq must be a DNA sequence or a number')
    if args.error_model.lower() in error_model_names:
        args.error_model = args.error_model.lower() if args.error_model.lower() == args.error_model else args.error_model
    if getattr(args, 'gpus', 1) < 1:
        sys.exit('Error: --gpus must be at least 1')
    if getattr(args, 'bam', False) and getattr(args, 'gzip', False):
        sys.exit('Error: --bam and --gzip cannot be used together (BAM is always compressed)')


def check_beta_identities(args):
    if args.mean_identity > 100.0:
        sys.exit('Error: mean read identity cannot be more than 100')
    if args.max_identity > 100.0:
        sys.exit('Error: max read identity cannot be more than 100')
    if args.mean_identity <= settings.MIN_MEAN_READ_IDENTITY:
        sys.exit(f'Error: mean read identity must be at least {settings.MIN_MEAN_READ_IDENTITY}')
    if args.max_identity <= settings.MIN_MEAN_READ_IDENTITY:
        sys.exit(f'Error: max read identity must be at least {settings.MIN_MEAN_READ_IDENTITY}')
    if args.mean_identity > args.max_identity:
        sys.exit(f'Error: mean identity ({args.mean_identity}) cannot be larger than max '
                 f'identity ({args.max_identity})')
    if args.identity_stdev < 0.0:
        sys.exit('Error: read identity stdev cannot be negative')


def check_qscore_identities(args):
    if args.mean_identity <= settings.MIN_MEAN_READ_QSCORE:
        sys.exit(f'Error: mean read identity must be at least {settings.MIN_MEAN_READ_QSCORE}')
    if args.identity_stdev < 0.0:
        sys.exit('Error: read qscore stdev cannot be negative')


if __name__ == '__main__':
    main()
