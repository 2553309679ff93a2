"""Compact storage of a nested fixture (dicts and lists of tensors and scalars) as one compressed ``.npz``.

Values that recur under the first list index of their path (the steps of a roll-out, the records of a
list) are stacked into one array, with the indices they came from where some items lack them, so a fixture
is a few dozen arrays rather than thousands of tiny ones.  ``load(save(x)) == x`` for tensors, ints,
floats, bools, strings, tuples of ints, and empty dicts / lists.
"""
import numpy as np
import torch


def _flatten(obj, path=()):
    if isinstance(obj, dict):
        if not obj:
            yield path, "ed", 0
        for k, v in obj.items():
            yield from _flatten(v, path + (("i" if isinstance(k, int) else "s") + str(k),))
    elif isinstance(obj, list):
        if not obj:
            yield path, "el", 0
        for i, v in enumerate(obj):
            yield from _flatten(v, path + ("l" + str(i),))
    elif isinstance(obj, torch.Tensor):
        yield path, "t", obj.detach().cpu().numpy()
    elif isinstance(obj, tuple):
        yield path, "u", np.array(obj, np.int64)
    elif isinstance(obj, bool):
        yield path, "b", obj
    elif isinstance(obj, int):
        yield path, "i", obj
    elif isinstance(obj, float):
        yield path, "f", obj
    elif isinstance(obj, str):
        yield path, "s", obj
    else:
        raise TypeError(f"{'/'.join(path)}: cannot store {type(obj).__name__}")


def save(path, obj):
    groups = {}
    for p, kind, value in _flatten(obj):
        lists = [n for n, c in enumerate(p) if c[0] == "l"]
        if lists and kind != "u":
            k = lists[0]
            template = "/".join(p[:k] + ("*",) + p[k + 1:])
            groups.setdefault((kind, template), []).append((int(p[k][1:]), value))
        else:
            groups.setdefault((kind, "/".join(p)), []).append((None, value))
    arrays = {}
    for (kind, template), items in groups.items():
        if items[0][0] is None:
            arrays[f"{kind}:{template}"] = np.asarray(items[0][1])
            continue
        values = [v for _, v in items]
        stackable = kind != "t" or all(v.shape == values[0].shape and v.dtype == values[0].dtype for v in values)
        if not stackable:  # one array per item
            for i, v in items:
                arrays[f"{kind}:{template.replace('*', 'l' + str(i), 1)}"] = v
            continue
        arrays[f"{kind}:{template}"] = np.stack(values) if kind == "t" else np.array(values)
        index = [i for i, _ in items]
        if index != list(range(len(index))):
            arrays[f"{kind}:{template}#idx"] = np.array(index, np.int64)
    np.savez_compressed(path, **arrays)


def _value(kind, a):
    if kind == "t":
        return torch.from_numpy(np.array(a))
    if kind == "u":
        return tuple(int(v) for v in a)
    if kind == "ed":
        return {}
    if kind == "el":
        return []
    return {"b": bool, "i": int, "f": float, "s": str}[kind](a)


def _build(node):
    if not isinstance(node, dict) or not node:
        return node
    if all(k[0] == "l" for k in node):
        return [_build(node[k]) for k in sorted(node, key=lambda k: int(k[1:]))]
    return {(int(k[1:]) if k[0] == "i" else k[1:]): _build(v) for k, v in node.items()}


def load(path):
    root = {}

    def put(p, value):
        parts = p.split("/") if p else []
        if not parts:
            return value
        node = root
        for c in parts[:-1]:
            node = node.setdefault(c, {})
        node[parts[-1]] = value

    with np.load(path) as data:
        for key in data.files:
            if key.endswith("#idx"):
                continue
            kind, template = key.split(":", 1)
            a = data[key]
            if "*" not in template:
                put(template, _value(kind, a))
                continue
            index = data[key + "#idx"] if key + "#idx" in data.files else range(len(a))
            for n, i in enumerate(index):
                put(template.replace("*", "l" + str(int(i)), 1), _value(kind, a[n]))
    return _build(root)
