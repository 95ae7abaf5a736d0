"""From-spec Merkle proofs by generalized index (consensus-specs ssz/merkle-proofs.md) over tests/ssz_spec.py and
hashlib.  TEST INFRASTRUCTURE: the second implementation the device branches are checked against.

Sparse: a tree of limit 2^40 with n chunks costs O(n) hashes, the nodes past the chunks are zero hashes."""
from lighthouse_b200.ssz_schema import pack_bits, serialize
from tests.ssz_spec import ZERO, _h, hash_tree_root, is_basic, pack


class Tree:
    """merkleize(chunks, 2**depth); children[i] = (type, value) behind composite leaf i, which a path may enter."""

    def __init__(self, chunks, depth, children=None):
        self.chunks, self.depth, self.children = chunks, depth, children
        self.memo = {}

    def node(self, level, i):
        if (i << level) >= len(self.chunks):
            return ZERO[level]
        if level == 0:
            return self.chunks[i]
        key = (level, i)
        if key not in self.memo:
            self.memo[key] = _h(self.node(level - 1, 2 * i), self.node(level - 1, 2 * i + 1))
        return self.memo[key]


def _depth(limit):
    return max(limit - 1, 0).bit_length()


def expand(t, v):
    """-> (chunk tree, length mixed in or None) of value v of type t."""
    k = t[0]
    if k == "uint":
        return Tree(pack(serialize(t, v)), 0), None
    if k == "bytes":
        return Tree(pack(v), _depth((t[1] + 31) // 32)), None
    if k == "bytelist":
        return Tree(pack(v), _depth((t[1] + 31) // 32)), len(v)
    if k == "bitvector":
        return Tree(pack(pack_bits(v, False)), _depth((t[1] + 255) // 256)), None
    if k == "bitlist":
        return Tree(pack(pack_bits(v, False)), _depth((t[1] + 255) // 256)), len(v)
    if k in ("vector", "list"):
        et, limit = t[1], t[2]
        if is_basic(et):
            tree = Tree(pack(b"".join(serialize(et, e) for e in v)), _depth((limit * et[1] + 31) // 32))
        else:
            tree = Tree([hash_tree_root(et, e) for e in v], _depth(limit), [(et, e) for e in v])
        return tree, (len(v) if k == "list" else None)
    fields = t[1]
    return Tree([hash_tree_root(ft, v[name]) for name, ft in fields], _depth(len(fields)),
                [(ft, v[name]) for name, ft in fields]), None


class Prover:
    """compute_merkle_proof over one value; expanded subtrees are kept, so many proofs of one value stay cheap."""

    def __init__(self, t, v):
        self.t, self.v = t, v
        self.cache = {}

    def _expand(self, key, t, v):
        if key not in self.cache:
            self.cache[key] = expand(t, v)
        return self.cache[key]

    def root(self):
        return hash_tree_root(self.t, self.v)

    def proof(self, gindex):
        """The branch of `gindex`, bottom-up (the leaf's sibling first).  ValueError below a leaf."""
        if gindex < 1:
            raise ValueError("gindex 0")
        branch = []
        cur = ("obj", self.t, self.v, 1)
        g = 1
        for b in bin(gindex)[3:]:
            bit = int(b)
            if cur[0] == "obj":
                _, t, v, at = cur
                tree, length = self._expand(at, t, v)
                cur = ("mix", tree, length, at) if length is not None else ("tree", tree, tree.depth, 0, at)
            if cur[0] == "mix":
                _, tree, length, at = cur
                if bit:
                    branch.append(tree.node(tree.depth, 0))
                    cur = ("leaf",)
                else:
                    branch.append(length.to_bytes(32, "little"))
                    cur = ("tree", tree, tree.depth, 0, at)
                g = 2 * g + bit
                continue
            if cur[0] == "tree" and cur[2] > 0:
                _, tree, level, i, at = cur
                branch.append(tree.node(level - 1, 2 * i + 1 - bit))
                level, i = level - 1, 2 * i + bit
                g = 2 * g + bit
                if level == 0 and tree.children and i < len(tree.children):
                    cur = ("obj",) + tree.children[i] + (g,)
                else:
                    cur = ("tree", tree, level, i, at)
                continue
            raise ValueError(f"gindex {gindex}: below a leaf")
        return branch[::-1]

    def node(self, gindex):
        """The value of the node `gindex` names: the first sibling of its own sibling's branch."""
        return self.root() if gindex == 1 else self.proof(gindex ^ 1)[0]


def compute_merkle_proof(t, v, gindex):
    return Prover(t, v).proof(gindex)


def root_from_branch(leaf, branch, gindex):
    """The root a leaf and its branch fold to (spec calculate_merkle_root)."""
    node = leaf
    for k, sib in enumerate(branch):
        node = _h(sib, node) if (gindex >> k) & 1 else _h(node, sib)
    return node
