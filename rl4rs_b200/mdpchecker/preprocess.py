"""script/mdpchecker/preprocess.py, the rl4rs branch: the sessions of rl4rs_dataset_a.csv with at least 16 history items
as `sessionid items` lines (the last 16 history items, then the first 5 exposed ones) in rl4rs.csv.

    python -m rl4rs_b200.mdpchecker.preprocess rl4rs DIR

The other datasets' branches (lastfm, cikm2016, recsys15, movielens) need pandasql and downloads of their raw data."""
import sys

OTHER = ("lastfm", "cikm2016", "recsys15", "movielens")


def preprocess(dataset_file, dataset_dir, print_fn=print):
    for name in OTHER:
        if name in dataset_file:
            raise NotImplementedError("preprocessing of the %s dataset is not built (it needs pandasql and the raw "
                                      "%s download)" % (name, name))
    if 'rl4rs' not in dataset_file:
        return None
    data = open(dataset_dir + '/rl4rs_dataset_a.csv', 'r').read().split('\n')[:-1]
    tmp = ['sessionid items']
    for x in data:
        f = x.split('@')
        session_id = f[1]
        sequence_id = list(map(int, f[5].split(',')))
        items = list(map(int, f[3].split(',')))
        if len(sequence_id) >= 16:
            tmp.append(session_id + ' ' + ','.join(list(map(str, sequence_id[-16:] + items[:5]))))
    print_fn('items num.', 283)
    print_fn('max item id', 283)
    print_fn('sessionid num.', len(tmp))
    out = dataset_dir + '/rl4rs.csv'
    with open(out, 'w') as f:
        f.write('\n'.join(tmp))
    return out


if __name__ == "__main__":
    preprocess(sys.argv[1], sys.argv[2])
