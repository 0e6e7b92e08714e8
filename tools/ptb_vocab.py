"""The reference's Penn Treebank word handling (main.py:44-59), shared by tools/train_ptb.py and tools/generate.py:
a file is read without its first character and split on single spaces; the vocabulary is the sorted set of the
training split's words, a word's id its index in that order."""
import os


def read_words(root, name):
    with open(os.path.join(root, name)) as f:
        return f.read()[1:].split(" ")


def vocabulary(train_words):
    """words (id -> word) and w2i (word -> id) from the training split's words."""
    words = sorted(set(train_words))
    return words, {w: i for i, w in enumerate(words)}
