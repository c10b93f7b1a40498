"""BASELINE.json configs[0] ("plumbing only"): the reference's basic usage with the import switched.

    python examples/basic_usage.py /path/to/local/bert-checkpoint      # any BERT/RoBERTa/DistilBERT-shaped HF directory

No network is needed: pass a local checkpoint directory (tests/test_gpu_classifier.py fabricates one from
tests/golden/golden_classifier.npz).  Needs an H100; there is no CPU fallback.
"""
import sys

from adaptive_classifier_b200 import AdaptiveClassifier   # was: from adaptive_classifier import AdaptiveClassifier


def main(model_dir: str):
    clf = AdaptiveClassifier(model_dir)                     # device defaults to "cuda"
    texts = ["the cat purrs on the sofa", "a kitten chases the yarn", "my cat sleeps all day", "cats love warm windows",
             "the tabby cat meows", "the dog barks at the mailman", "a puppy fetches the stick", "my dog loves long walks",
             "dogs wag their tails", "the beagle howls at night"]
    labels = ["cat"] * 5 + ["dog"] * 5
    clf.add_examples(texts, labels)
    for t in ("a cat naps in the sun", "the dog runs in the park"):
        print(t, "->", clf.predict(t, k=2))
    print(clf.predict_batch(["kittens and cats", "puppies and dogs"], k=1))
    clf.save("./cat_dog_classifier")
    again = AdaptiveClassifier.load("./cat_dog_classifier")
    print("reloaded:", again.predict("a cat naps in the sun", k=2))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "bert-base-uncased")
