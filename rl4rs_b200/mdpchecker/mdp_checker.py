"""script/mdpchecker/mdp_checker.py: fit the seq2seq transformer on a logged dataset, then beam-search held-out rows and
print Experiment II (score ratios of the greedy, top and hot beams) and Experiment I (how well each prefix's probability
predicts the whole path's: Pearson and Spearman).

    python -m rl4rs_b200.mdpchecker.mdp_checker NAME DIR

reads DIR/NAME.csv (`sessionid items` lines, as preprocess writes them) and prints the script's lines.  The weights go to
NAME.npz in the working directory (the script writes NAME.h5)."""
import random
import sys
import warnings

import numpy as np
from scipy.stats import spearmanr

from rl4rs_b200.mdpchecker.decoder import beam_search, path_probs
from rl4rs_b200.mdpchecker.transformer import get_model


def prepare(dataset_file, dataset_dir, print_fn=print):
    """The script's data preparation, up to `# Build & fit model`: the window rule and its np.random draws, the token
    dicts, START / END / PAD and the padding.  Returns (encode_input, decode_input, decode_output, source_token_dict,
    target_token_dict, target_len)."""
    if 'recsys15' in dataset_file:
        source_len = 8
    elif 'cikm2016' in dataset_file:
        source_len = 5
    else:
        source_len = 16
    target_len = 5
    np.random.seed(1)
    data = open(dataset_dir + '/' + dataset_file).read().split('\n')[1:-1]
    source_tokens, target_tokens = [], []
    for sample in data:
        user_id, items = sample.split(' ')
        item_list = items.split(',')
        if len(item_list) >= source_len + target_len:
            i = 0
            if 'rl4rs' in dataset_file or 'cikm2016' in dataset_file:
                source_tokens.append(item_list[:source_len])
                target_tokens.append(item_list[source_len:source_len + target_len])
            else:
                while i + source_len + target_len < len(item_list):
                    source_tokens.append(item_list[i: i + source_len])
                    target_tokens.append(item_list[i + source_len: i + source_len + target_len])
                    i = i + np.random.randint(source_len, source_len + target_len) // 6
        else:
            print_fn('len(item_list) <= source_len + target_len in', '\t', sample)

    # one dict grows through both token lists, as in the script (the target dict is the same object)
    token_dict = {'<PAD>': 0, '<START>': 1, '<END>': 2}

    def build_token_dict(token_list):
        for tokens in token_list:
            for token in tokens:
                if token not in token_dict:
                    token_dict[token] = len(token_dict)
        return token_dict

    source_token_dict = build_token_dict(source_tokens)
    target_token_dict = build_token_dict(target_tokens)
    encode_tokens = [['<START>'] + tokens + ['<END>'] for tokens in source_tokens]
    decode_tokens = [['<START>'] + tokens + ['<END>'] for tokens in target_tokens]
    output_tokens = [tokens + ['<END>', '<PAD>'] for tokens in target_tokens]
    source_max_len = max(map(len, encode_tokens))
    target_max_len = max(map(len, decode_tokens))
    encode_tokens = [tokens + ['<PAD>'] * (source_max_len - len(tokens)) for tokens in encode_tokens]
    decode_tokens = [tokens + ['<PAD>'] * (target_max_len - len(tokens)) for tokens in decode_tokens]
    output_tokens = [tokens + ['<PAD>'] * (target_max_len - len(tokens)) for tokens in output_tokens]
    encode_input = [list(map(lambda x: source_token_dict[x], tokens)) for tokens in encode_tokens]
    decode_input = [list(map(lambda x: target_token_dict[x], tokens)) for tokens in decode_tokens]
    decode_output = [list(map(lambda x: [target_token_dict[x]], tokens)) for tokens in output_tokens]
    print_fn('sample lens:', len(encode_input))
    print_fn('source_token_dict lens:', len(source_token_dict))
    print_fn('target_token_dict lens:', len(target_token_dict))
    return encode_input, decode_input, decode_output, source_token_dict, target_token_dict, target_len


def experiment_one(probs):
    """Experiment I's table [5, 2] (mean over rows of Pearson / Spearman between each prefix's product of probabilities
    and the whole path's), from probs [n, beam, 5]; NaN (a constant input) counts as 1.0, as in the script."""
    n = probs.shape[0]
    metrics = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for j in range(n):
            prob = probs[j]
            seq_score = np.multiply.reduce(np.array(prob), axis=1)
            for i in range(5):
                part = np.multiply.reduce(np.array(prob[:, :i + 1]), axis=1)
                metrics.append((np.corrcoef(part, seq_score)[0][1], spearmanr(part, seq_score)[0]))
    metrics = np.array(metrics).reshape((n, 5, 2))
    metrics = np.nan_to_num(metrics, nan=1.0)
    return np.nanmean(metrics, axis=0)


def main(dataset, dataset_dir, epochs=20, holdout=10000, eval_rows=2048, beam_size=100, embed_dim=256, hidden_dim=128,
         batch_size=256, weights_path=None, seed=0, device=None, print_fn=print):
    """The script's flow; its defaults are the script's.  Returns the printed numbers: 'experiment_ii' (the five ratios),
    'experiment_i' ([5, 2]), and the searches' outputs."""
    dataset_file = dataset + '.csv'
    encode_input, decode_input, decode_output, source_token_dict, target_token_dict, target_len = prepare(
        dataset_file, dataset_dir, print_fn)
    model = get_model(
        token_num=max(len(source_token_dict), len(target_token_dict)),
        embed_dim=embed_dim,
        encoder_num=1,
        decoder_num=1,
        head_num=1,
        hidden_dim=hidden_dim,
        dropout_rate=0.05,
        use_same_embed=False,
        seed=seed,
        device=device,
    )
    model.compile('adam', 'sparse_categorical_crossentropy')
    model.summary(print_fn=print_fn)
    history = model.fit(
        x=[np.array(encode_input)[:-holdout], np.array(decode_input)[:-holdout]],
        y=np.array(decode_output)[:-holdout],
        epochs=epochs,
        batch_size=batch_size,
        shuffle=True,
        verbose=2,
        print_fn=print_fn,
    )
    weights_path = weights_path or dataset_file.split('.')[0] + '.npz'
    model.save_weights(weights_path)
    model.load_weights(weights_path)

    batch = eval_rows
    hot_beam_size = 20 if 'rl4rs' in dataset_file else beam_size
    candidates_size = 6000 if 'cikm2016' in dataset_file else hot_beam_size
    random.seed(1)
    encode_input = random.sample(encode_input[-holdout:], batch)
    output_greedy, greedy_score = beam_search(model, encode_input, beam_size=1, target_len=target_len)
    output_topk, beam_score = beam_search(model, encode_input, beam_size=beam_size, target_len=target_len)
    beam_score_5 = beam_score[:, :int(beam_size * 0.05)]
    beam_score_20 = beam_score[:, :int(beam_size * 0.2)]
    output_topk_hot, beam_score_hot = beam_search(model, encode_input, beam_size=hot_beam_size, target_len=target_len,
                                                  use_candidates=True, candidates_size=candidates_size)
    beam_score_hot5 = beam_score_hot[:, :int(beam_size * 0.05)]
    beam_score_hot20 = beam_score_hot[:, :int(beam_size * 0.2)]

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        greedy = np.nanmean(greedy_score, axis=1)
        top5 = np.nanmean(beam_score_5, axis=1)
        top20 = np.nanmean(beam_score_20, axis=1)
        hot5 = np.nanmean(beam_score_hot5, axis=1)
        hot20 = np.nanmean(beam_score_hot20, axis=1)
        exp2 = [1, np.nanmean(top20 / top5), np.nanmean(greedy / top5), np.nanmean(hot5 / top5), np.nanmean(hot20 / top5)]
    print_fn('experiment II results')
    print_fn('top_5_percent_score top_20_percent_score greedy_score hot_5_percent_score hot_20_percent_score')
    print_fn(*exp2)

    print_fn('experiment I start')
    exp1 = experiment_one(path_probs(model, encode_input, output_topk)[:, :, :5])
    print_fn('experiment I results')
    print_fn('corrcoef', ' ', 'spearman')
    print_fn(exp1)
    return {"experiment_ii": exp2, "experiment_i": exp1, "output_greedy": output_greedy, "greedy_score": greedy_score,
            "output_topk": output_topk, "beam_score": beam_score, "output_topk_hot": output_topk_hot,
            "beam_score_hot": beam_score_hot, "encode_input": encode_input, "loss": history.history["loss"],
            "model": model}


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
