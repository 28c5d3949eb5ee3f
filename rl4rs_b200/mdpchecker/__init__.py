"""The MDP checker (the paper's data-understanding tool): a seq2seq transformer fitted on logged sequences, then beam
searches whose scores tell whether the data behaves like an MDP.  `transformer.get_model`, `decoder`, `preprocess` and
`mdp_checker` carry the reference's names."""
